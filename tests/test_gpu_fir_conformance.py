"""The FIR resampling and glue kernels of engine.cu against an fp64 reference, over a table of launches that reaches every kernel and
tile configuration their entry points can select:

    n3d_fir_up_epilogue   fir_up_stream_kernel (TR 32 / 64 / 128) or fir_up_epilogue_kernel (strip length S)
    n3d_fir_down_split    fir_down_stream_kernel (TS 16 / 32) or fir_down_split_kernel (strip length S)
    n3d_splitk_epilogue   splitk_epilogue_kernel
    n3d_modulate_split    modulate_split_kernel
    n3d_upsample2d_nhwc   upsample2d_kernel<4> or <1>
    n3d_downsample2d_nhwc downsample2d_kernel

The references are oracle.ops (upfirdn2d / upsample2d / downsample2d) evaluated in fp64 on the device, followed by the mode-0 epilogue
in fp64.  They are computed one image and at most REF_CHANNELS channels at a time, so that the largest launches (which the streamed
TR 128 tile and the S 16 strips need) stay within about 512 MB including their reference.

Every output is a view into a larger allocation filled with a NaN sentinel: the elements a launch owns must be written (and match),
every other element -- guard bands, the other half of a concat buffer, channels outside [coff, coff + C) -- must keep the sentinel's
bits.  Each case is then rerun as it is, and a case that takes a streamed kernel is rerun under N3D_FIR_STREAM=0 (the register-tiled
kernels everywhere): both reruns must be bit-identical.

`fir_up_plan` / `fir_down_plan` mirror the launch rules in plain Python.  The CPU test checks that the table covers everything in
COVERAGE; the profiler test checks on the GPU that each case ran the kernel (and grid) the plan predicts.  The alignment tests at the
end need no GPU: misaligned host pointers must be refused before any device call.
"""
import math
import re

import pytest
import torch
import torch.nn.functional as F

from tests.helpers import Guarded, RangeErr, cdiv, grid_stride, launched_kernels, lib, offset_view, record_errors, refused, rerun_identical

DEV = 'cuda'
SMS = 132                   # SM count the table is planned at (H100 SXM)
REF_CHANNELS = 16           # channels per fp64 reference chunk
SQRT2 = math.sqrt(2.0)

# Range-relative error bounds, max |got - ref| / max |ref| over the owned elements of an output, each at most 4x the worst case
# measured over the table on an H100 80GB HBM3 (400 W power limit), which is given beside it.  N3D_FIR_ERRORS=<file> appends every
# measured error to that file as JSON lines.
BOUNDS = {
    'up.f32': 2e-6,         # fir-up epilogue, fp32 output.  Worst: 5.5e-7 (up_stream_c64_tr128)
    'up.split': 2.5e-5,     # fir-up epilogue, hi + lo of a split output (the split rounds at 2^-17 of the value).  Worst: 6.6e-6 (up_tiled_c12)
    'splitk.f32': 9e-7,     # Worst: 2.3e-7 (splitk_s9: 9 partial sums)
    'splitk.split': 2e-5,   # Worst: 5.1e-6 (splitk_s1)
    'down.split': 2e-5,     # fir-down, hi + lo of the four parity images.  Worst: 5.3e-6 (down_stream_c256_h2)
    'modsplit.split': 2e-5,     # Worst: 5.1e-6 (modsplit_grid)
    'upsample': 4e-7,       # Worst: 1.0e-7 (upsample_c3_nchw_grid)
    'downsample': 7.5e-7,   # Worst: 1.9e-7 (downsample_c32_grid)
}


# ------------------------------------------------------------------------------------------------ the launch rules, mirrored
def fir_strip_rows(sms, threads_per_row, rows):
    """fir_strip_rows (engine.cu): 16 rows per strip, halved down to 4 while the launch has < 1024 threads per SM, clipped to rows."""
    S = 16
    while S > 4 and threads_per_row * cdiv(rows, S) < sms * 1024:
        S >>= 1
    return min(S, rows)


def fir_up_plan(N, H2, W2, C, sms=SMS):
    """n3d_fir_up_epilogue: streamed when TC = 2048 / C (64 <= C <= 512) divides W2 and some TR in {32, 64, 128} dividing H2 gives
    >= sms CTAs (the one with the best last-wave fill x (1 - vertical halo), first on ties); otherwise the register-tiled kernel."""
    TC = 2048 // C if 64 <= C <= 512 and 2048 % C == 0 else 0
    TR, best = 0, 0.0
    if TC >= 4 and W2 % TC == 0:
        for tr in (32, 64, 128):
            if H2 % tr:
                continue
            ctas = N * (W2 // TC) * (H2 // tr)
            if ctas < sms:
                continue
            eff = ctas / (cdiv(ctas, 2 * sms) * 2 * sms) * tr / (tr + 3)
            if eff > best:
                best, TR = eff, tr
    if TR:
        return dict(kernel='fir_up_stream_kernel', streamed=True, TC=TC, TR=TR, grid=N * (W2 // TC) * (H2 // TR))
    why = ('channels' if not TC else 'width' if W2 % TC else 'height' if all(H2 % tr for tr in (32, 64, 128)) else 'ctas')
    S = fir_strip_rows(sms, N * (W2 // 2) * (C // 4), H2 // 2)
    total = N * cdiv(H2 // 2, S) * (W2 // 2) * (C // 4)
    return dict(kernel='fir_up_epilogue_kernel', streamed=False, S=S, rows=H2 // 2, why=why, work=total, grid=grid_stride(total, sms, 16))


def fir_down_plan(N, H, W, C, sms=SMS):
    """n3d_fir_down_split: streamed when TSC = 256 / (C / 4) (8 <= C / 4 <= 128) and TS = 32, else 16, gives >= sms CTAs; otherwise
    the register-tiled kernel."""
    c4n, SH, SW = C // 4, (H + 2) // 2, (W + 2) // 2
    TSC = 256 // c4n if 8 <= c4n <= 128 and 256 % c4n == 0 else 0
    for ts in (32, 16):
        if TSC and N * cdiv(SW, TSC) * cdiv(SH, ts) >= sms:
            return dict(kernel='fir_down_stream_kernel', streamed=True, TSC=TSC, TS=ts, ragged_rows=SH % ts != 0, ragged_cols=SW % TSC != 0,
                        grid=N * cdiv(SW, TSC) * cdiv(SH, ts))
    S = fir_strip_rows(sms, N * SW * c4n, SH)
    total = N * cdiv(SH, S) * SW * c4n
    return dict(kernel='fir_down_split_kernel', streamed=False, S=S, rows=SH, work=total, grid=grid_stride(total, sms, 16))


def upsample2d_vec(C):
    """n3d_upsample2d_nhwc: 4 channels per thread when C % 4 == 0 (and the pointers are 16-byte aligned, as every case's are)."""
    return 4 if C % 4 == 0 else 1


def plan(c, sms=SMS):
    """Kernel, grid and grid-stride work items of a case."""
    k, N, H, W, Cc = c['kind'], c['N'], c['H'], c['W'], c['C']
    if k == 'up':
        return fir_up_plan(N, H, W, Cc, sms)
    if k == 'down':
        return fir_down_plan(N, H, W, Cc, sms)
    if k == 'upsample':
        v = upsample2d_vec(Cc)
        work = N * H * W * Cc // v
        return dict(kernel=f'upsample2d_kernel<{v}>', streamed=False, work=work, grid=grid_stride(work, sms, 16))
    work = {'downsample': N * (H // 2) * (W // 2) * Cc, 'splitk': N * H * W * Cc // 4, 'modsplit': N * H * W * Cc // 4}[k]
    name = {'downsample': 'downsample2d_kernel', 'splitk': 'splitk_epilogue_kernel', 'modsplit': 'modulate_split_kernel'}[k]
    return dict(kernel=name, streamed=False, work=work, grid=grid_stride(work, sms, 16))


# ------------------------------------------------------------------------------------------------ the case table
def _case(name, kind, N, H, W, Cc, **kw):
    """H, W: output size of the epilogue kinds ('up', 'splitk'), input size of the others.  outs: split outputs (cstride, coff,
    style); f32: the fp32 output (cstride, coff) or None.  Epilogue: dcoef / bias present, gain, slope, clamp (< 0: off), noise."""
    c = dict(name=name, kind=kind, N=N, H=H, W=W, C=Cc, dcoef=True, bias=True, gain=SQRT2, slope=0.2, clamp=-1.0, noise='shared',
             outs=[], f32=dict(cstride=Cc, coff=0), S=1, nchw=False)
    c.update(kw)
    return c


def _out(cstride, coff=0, style=True):
    return dict(cstride=cstride, coff=coff, style=style)


PLAIN = dict(dcoef=False, bias=False, gain=1.0, slope=1.0, clamp=-1.0, noise='none')     # conv2d_resample's form of the epilogue
CASES = [
    # fir-up, streamed: every C of the streamed set, every TR
    _case('up_stream_c64_tr128', 'up', 5, 512, 320, 64, noise='sample', clamp=2.0),
    _case('up_stream_c512_tr32', 'up', 1, 32, 528, 512, noise='sample', f32=None, outs=[_out(512), _out(1024, 512, style=False)]),
    _case('up_stream_c256_tr64', 'up', 1, 448, 152, 256, clamp=2.0, f32=dict(cstride=264, coff=8), outs=[_out(256)]),
    _case('up_stream_c128_tr32_plain', 'up', 1, 128, 528, 128, **PLAIN),
    # fir-up, register-tiled: C outside the streamed set, W2 % TC != 0, H2 not a multiple of 32, too few CTAs
    _case('up_tiled_c12', 'up', 2, 18, 10, 12, noise='sample', clamp=1.0, f32=None, outs=[_out(12), _out(24, 12)]),
    _case('up_tiled_c96', 'up', 2, 40, 24, 96, f32=dict(cstride=100, coff=4), outs=[_out(96, style=False)]),
    _case('up_tiled_width_plain', 'up', 2, 64, 40, 128, **PLAIN),
    _case('up_tiled_height', 'up', 3, 48, 64, 64, noise='none', clamp=2.0, outs=[_out(64)]),
    _case('up_tiled_ctas', 'up', 1, 64, 64, 256, gain=1.0, noise='sample'),
    # fir-up strips: S 16 and 8, S clipped below 4 (H2 = 2 and 6, the latter 2 pixels wide)
    _case('up_tiled_s16', 'up', 4, 256, 264, 128),
    _case('up_tiled_s8', 'up', 2, 256, 264, 128, f32=None, outs=[_out(128)], clamp=2.0),
    _case('up_tiled_h2', 'up', 3, 2, 8, 16, noise='sample', outs=[_out(32, 16)]),
    _case('up_tiled_h6_w2', 'up', 2, 6, 2, 8, slope=1.0, clamp=0.5, outs=[_out(8, style=False)]),
    # split-K epilogue: S 1, 2, 9
    _case('splitk_s1', 'splitk', 2, 8, 12, 16, S=1, noise='sample', clamp=2.0, f32=None, outs=[_out(16), _out(32, 16)]),
    _case('splitk_s2_plain_grid', 'splitk', 2, 64, 64, 320, S=2, **PLAIN),
    _case('splitk_s9', 'splitk', 3, 4, 6, 64, S=9, clamp=2.0, gain=1.0, f32=dict(cstride=72, coff=8), outs=[_out(64, style=False)]),
    # modulate_split
    _case('modsplit_style', 'modsplit', 2, 5, 7, 16, outs=[_out(24, 8)]),
    _case('modsplit_nostyle', 'modsplit', 3, 4, 6, 8, outs=[_out(8, style=False)]),
    _case('modsplit_grid', 'modsplit', 2, 64, 72, 256, outs=[_out(256)]),
    # upsample2d / downsample2d
    _case('upsample_c3_nchw', 'upsample', 2, 7, 12, 3, nchw=True),
    _case('upsample_c1_h1', 'upsample', 3, 1, 9, 1),
    _case('upsample_c32', 'upsample', 2, 5, 8, 32),
    _case('upsample_c32_nchw', 'upsample', 1, 6, 4, 32, nchw=True),
    _case('upsample_c3_nchw_grid', 'upsample', 4, 200, 240, 3, nchw=True),
    _case('downsample_c3', 'downsample', 2, 6, 10, 3),
    _case('downsample_c32', 'downsample', 3, 8, 14, 32),
    _case('downsample_c32_grid', 'downsample', 4, 128, 140, 32),
    # fir-down, streamed: every C of the streamed set, TS 16 and 32, ragged and exact last tiles
    _case('down_stream_c32', 'down', 8, 190, 128, 32),
    _case('down_stream_c64_ts32', 'down', 7, 254, 128, 64),
    _case('down_stream_c128_ragged', 'down', 6, 32, 160, 128),
    _case('down_stream_c256_h2', 'down', 6, 2, 168, 256),
    _case('down_stream_c512_exact', 'down', 8, 286, 6, 512),
    # fir-down, register-tiled: C 4, 24, 96; S 16, 8, a ragged S 4, S clipped below 4; 2 pixels wide
    _case('down_tiled_c96_s16', 'down', 8, 190, 254, 96),
    _case('down_tiled_c96_s8', 'down', 4, 190, 254, 96),
    _case('down_tiled_c24_s4', 'down', 2, 20, 14, 24),
    _case('down_tiled_c4', 'down', 3, 8, 12, 4),
    _case('down_tiled_w2', 'down', 2, 10, 2, 24),
    _case('down_tiled_h2', 'down', 2, 2, 6, 8),
]
CASE_IDS = [c['name'] for c in CASES]
_EPI = ('up', 'splitk')


def _epi_cover(kind):
    """COVERAGE items of one epilogue entry point."""
    k = lambda cs: [c for c, p in cs if c['kind'] == kind]                   # noqa: E731
    return {
        f'{kind}: dcoef and bias present and absent': lambda cs: {(c['dcoef'], c['bias']) for c in k(cs)} >= {(True, True), (False, False)},
        f'{kind}: slope 0.2 and 1': lambda cs: {c['slope'] for c in k(cs)} >= {0.2, 1.0},
        f'{kind}: gain sqrt 2 and 1': lambda cs: {c['gain'] for c in k(cs)} >= {SQRT2, 1.0},
        f'{kind}: clamp off and on': lambda cs: {c['clamp'] >= 0 for c in k(cs)} == {False, True},
        f'{kind}: noise none, shared, per sample': lambda cs: {c['noise'] for c in k(cs)} == {'none', 'shared', 'sample'},
        f'{kind}: 0, 1 and 2 split outputs': lambda cs: {len(c['outs']) for c in k(cs)} == {0, 1, 2},
        f'{kind}: a split output without style': lambda cs: any(not o['style'] for c in k(cs) for o in c['outs']),
        f'{kind}: a split output into the second half of a concat buffer':
            lambda cs: any(o['coff'] == c['C'] and o['cstride'] == 2 * c['C'] for c in k(cs) for o in c['outs']),
        f'{kind}: no fp32 output': lambda cs: any(c['f32'] is None for c in k(cs)),
        f'{kind}: fp32 output at cstride > C, coff > 0': lambda cs: any(c['f32'] and c['f32']['cstride'] > c['C'] and c['f32']['coff'] > 0 for c in k(cs)),
    }


def _planned(kind, cs):
    return [(c, p) for c, p in cs if c['kind'] == kind]


COVERAGE = {
    'fir-up streamed at C 64, 128, 256, 512': lambda cs: {c['C'] for c, p in _planned('up', cs) if p['streamed']} == {64, 128, 256, 512},
    'fir-up streamed at TR 32, 64, 128': lambda cs: {p['TR'] for c, p in _planned('up', cs) if p['streamed']} == {32, 64, 128},
    'fir-up register-tiled for every reason': lambda cs: {p['why'] for c, p in _planned('up', cs) if not p['streamed']} == {'channels', 'width', 'height', 'ctas'},
    'fir-up register-tiled at C 12 and 96': lambda cs: {c['C'] for c, p in _planned('up', cs) if not p['streamed']} >= {12, 96},
    'fir-up strips S 16, 8, 4': lambda cs: {p['S'] for c, p in _planned('up', cs) if not p['streamed']} >= {16, 8, 4},
    'fir-up ragged last strip': lambda cs: any(not p['streamed'] and p['rows'] % p['S'] for c, p in _planned('up', cs)),
    'fir-up strips clipped below 4 rows (H2 2 and 6)': lambda cs: {c['H'] for c, p in _planned('up', cs) if not p['streamed'] and p['S'] < 4} >= {2, 6},
    'fir-down streamed at C 32, 64, 128, 256, 512': lambda cs: {c['C'] for c, p in _planned('down', cs) if p['streamed']} == {32, 64, 128, 256, 512},
    'fir-down streamed at TS 16 and 32': lambda cs: {p['TS'] for c, p in _planned('down', cs) if p['streamed']} == {16, 32},
    'fir-down streamed with ragged and exact last row tiles': lambda cs: {p['ragged_rows'] for c, p in _planned('down', cs) if p['streamed']} == {False, True},
    'fir-down streamed with ragged and exact last column tiles': lambda cs: {p['ragged_cols'] for c, p in _planned('down', cs) if p['streamed']} == {False, True},
    'fir-down register-tiled at C 4, 24, 96': lambda cs: {c['C'] for c, p in _planned('down', cs) if not p['streamed']} >= {4, 24, 96},
    'fir-down strips S 16, 8, 4': lambda cs: {p['S'] for c, p in _planned('down', cs) if not p['streamed']} >= {16, 8, 4},
    'fir-down ragged strip of 4': lambda cs: any(not p['streamed'] and p['S'] == 4 and p['rows'] % 4 for c, p in _planned('down', cs)),
    'fir-down strips clipped below 4 rows': lambda cs: any(not p['streamed'] and p['S'] < 4 for c, p in _planned('down', cs)),
    'H != W on both FIR kernels in both forms': lambda cs: {(c['kind'], p['streamed']) for c, p in cs if c['kind'] in ('up', 'down') and c['H'] != c['W']}
        == {('up', False), ('up', True), ('down', False), ('down', True)},
    '2-pixel-wide image on both FIR kernels': lambda cs: {c['kind'] for c, p in cs if c['kind'] in ('up', 'down') and c['W'] == 2} == {'up', 'down'},
    **_epi_cover('up'),
    **_epi_cover('splitk'),
    'split-K with S 1, 2, 9': lambda cs: {c['S'] for c, p in _planned('splitk', cs)} >= {1, 2, 9},
    'modulate_split with and without style': lambda cs: {o['style'] for c, p in _planned('modsplit', cs) for o in c['outs']} == {False, True},
    'modulate_split at a channel offset': lambda cs: any(o['coff'] > 0 for c, p in _planned('modsplit', cs) for o in c['outs']),
    'upsample2d at C 3, 1, 32': lambda cs: {c['C'] for c, p in _planned('upsample', cs)} >= {1, 3, 32},
    'upsample2d both kernels': lambda cs: {p['kernel'] for c, p in _planned('upsample', cs)} == {'upsample2d_kernel<4>', 'upsample2d_kernel<1>'},
    'upsample2d NHWC and NCHW output': lambda cs: {c['nchw'] for c, p in _planned('upsample', cs)} == {False, True},
    'upsample2d H != W and H 1': lambda cs: any(c['H'] != c['W'] for c, p in _planned('upsample', cs)) and any(c['H'] == 1 for c, p in _planned('upsample', cs)),
    'downsample2d at C 3 and 32, H != W': lambda cs: {c['C'] for c, p in _planned('downsample', cs) if c['H'] != c['W']} >= {3, 32},
    'grid-stride loop of modulate_split, upsample2d, downsample2d, splitk_epilogue':
        lambda cs: {c['kind'] for c, p in cs if 'work' in p and p['work'] > p['grid'] * 256} >= {'modsplit', 'upsample', 'downsample', 'splitk'},
}


def case_bytes(c):
    """Device memory of a case: inputs, guarded outputs, and four fp64 tensors the size of one reference chunk (the copies
    upfirdn2d and the epilogue make)."""
    N, H, W, Cc, k = c['N'], c['H'], c['W'], c['C'], c['kind']
    chunk = 4 * (H + 4) * (W + 4) * min(Cc, REF_CHANNELS) * 8
    if k in _EPI:
        inp = N * (H + 1) * (W + 1) * Cc * 4 if k == 'up' else c['S'] * N * H * W * Cc * 4
        outs = sum(2 * N * H * W * o['cstride'] * 2 for o in c['outs']) + (N * H * W * c['f32']['cstride'] * 4 if c['f32'] else 0)
    elif k == 'down':
        inp, outs = N * H * W * Cc * 4, 2 * 4 * N * (H // 2 + 1) * (W // 2 + 1) * Cc * 2
    elif k == 'modsplit':
        inp, outs = N * H * W * Cc * 4, 2 * N * H * W * c['outs'][0]['cstride'] * 2
    else:
        inp = N * H * W * Cc * 4
        outs = inp * 4 if k == 'upsample' else inp // 4
        chunk = max(chunk, 4 * outs // N * 2)
    return inp + outs + chunk


def test_case_table_covers_every_launch_configuration():
    """CPU: the table reaches everything listed in COVERAGE, according to the mirrored launch rules, at <= 512 MB per case."""
    planned = [(c, plan(c)) for c in CASES]
    missing = [k for k, ok in COVERAGE.items() if not ok(planned)]
    assert not missing, missing
    assert len(set(CASE_IDS)) == len(CASE_IDS)
    big = {c['name']: case_bytes(c) / 2 ** 20 for c in CASES if case_bytes(c) > 512 * 2 ** 20}
    assert not big, big


# ------------------------------------------------------------------------------------------------ outputs and inputs
def _seeded(c):
    return torch.Generator(device=DEV).manual_seed(2000 + CASE_IDS.index(c['name']))


def setup_case(c):
    """Inputs and guarded outputs of a case (the device tensors every launch points at)."""
    g = _seeded(c)
    N, H, W, Cc, k = c['N'], c['H'], c['W'], c['C'], c['kind']
    s = dict(c=c, outs=[], f32=None)
    rnd = lambda *shape: torch.randn(*shape, device=DEV, generator=g)      # noqa: E731
    if k in _EPI:
        s['x'] = rnd(N, H + 1, W + 1, Cc) if k == 'up' else rnd(c['S'], N, H, W, Cc) / math.sqrt(c['S'])
        s['dcoef'] = torch.rand(N, Cc, device=DEV, generator=g) + 0.5 if c['dcoef'] else None
        s['bias'] = rnd(Cc) * 0.5 if c['bias'] else None
        s['noise'] = {'none': None, 'shared': rnd(H, W) * 0.3, 'sample': rnd(N, H, W) * 0.3}[c['noise']]
        s['noise_nstride'] = H * W if c['noise'] == 'sample' else 0
    else:
        s['x'] = rnd(N, H, W, Cc)
    if k in _EPI or k == 'modsplit':
        for o in c['outs']:
            hi, lo = (Guarded((N, H, W, o['cstride']), torch.bfloat16, slice(o['coff'], o['coff'] + Cc)) for _ in range(2))
            s['outs'].append((hi, lo, rnd(N, Cc) if o['style'] else None))
    if k in _EPI and c['f32']:
        f = c['f32']
        s['f32'] = Guarded((N, H, W, f['cstride']), torch.float32, slice(f['coff'], f['coff'] + Cc))
    if k == 'down':
        SH, SW = (H + 2) // 2, (W + 2) // 2
        s['outs'] = [(Guarded((4, N, SH, SW, Cc), torch.bfloat16), Guarded((4, N, SH, SW, Cc), torch.bfloat16), None)]
    if k in ('upsample', 'downsample'):
        OH, OW = (2 * H, 2 * W) if k == 'upsample' else (H // 2, W // 2)
        s['f32'] = Guarded((N, Cc, OH, OW) if c['nchw'] else (N, OH, OW, Cc), torch.float32)
    return s


def outputs(s):
    return [t for hi, lo, _ in s['outs'] for t in (hi, lo)] + ([s['f32']] if s['f32'] is not None else [])


def launch_case(s):
    from next3d_b200 import kernels as K
    c = s['c']
    k = c['kind']
    if k in _EPI:
        outs = [K.make_split_out(hi.view, lo.view, sty, o['cstride'], o['coff']) for (hi, lo, sty), o in zip(s['outs'], c['outs'])]
        f = c['f32'] or dict(cstride=0, coff=0)
        fn = K.fir_up_epilogue if k == 'up' else K.splitk_epilogue
        args = (s['x'], c['C']) if k == 'up' else (s['x'],)
        fn(*args, s['dcoef'], s['bias'], s['noise'], c['gain'], c['slope'], c['clamp'], outs=outs,
           out_f32=s['f32'].view if s['f32'] else None, f32_cstride=f['cstride'], f32_coff=f['coff'], noise_nstride=s['noise_nstride'])
    elif k == 'modsplit':
        (hi, lo, sty), o = s['outs'][0], c['outs'][0]
        K.modulate_split(s['x'], sty, hi.view, lo.view, o['cstride'], o['coff'])
    elif k == 'down':
        hi, lo, _ = s['outs'][0]
        N, H, W, Cc = s['x'].shape
        K.fir_down_split(s['x'], hi.view.view(4 * N, (H + 2) // 2, (W + 2) // 2, Cc), lo.view.view(4 * N, (H + 2) // 2, (W + 2) // 2, Cc))
    elif k == 'upsample':
        K.upsample2d_nhwc(s['x'], s['f32'].view, y_nchw=c['nchw'])
    else:
        K.downsample2d_nhwc(s['x'], s['f32'].view)


# ------------------------------------------------------------------------------------------------ the fp64 reference
def _filter64():
    from oracle import ops as oo
    return oo.setup_filter().to(DEV, torch.float64)


def epilogue_reference(acc, s, n, c0, c1):
    """Mode-0 epilogue in fp64 of image n, channels [c0, c1): acc [H, W, c] -> v = acc * dcoef + noise + bias; lrelu_slope(v) * gain;
    clamp."""
    c = s['c']
    v = acc
    if s['dcoef'] is not None:
        v = v * s['dcoef'][n, c0:c1].double()
    if s['noise'] is not None:
        v = v + (s['noise'][n] if c['noise'] == 'sample' else s['noise']).double()[..., None]
    if s['bias'] is not None:
        v = v + s['bias'][c0:c1].double()
    v = torch.where(v > 0, v, v * c['slope']) * c['gain']
    if c['clamp'] >= 0:
        v = v.clamp(-c['clamp'], c['clamp'])
    return v


def _chunks(s):
    Cc = s['c']['C']
    for n in range(s['c']['N']):
        for c0 in range(0, Cc, REF_CHANNELS):
            yield n, c0, min(Cc, c0 + REF_CHANNELS)


def check_case(s):
    """-> {bound kind: range-relative error}; asserts the sentinel and written-element checks first."""
    from oracle import ops as oo
    c = s['c']
    k = c['kind']
    for t in outputs(s):
        assert t.untouched_ok(), f'{c["name"]}: an element outside the output was written'
        assert t.written(), f'{c["name"]}: an owned element was not written'
    errs = {}
    f64 = _filter64()
    if k in _EPI:
        e_f32, e_split = RangeErr(), [RangeErr() for _ in s['outs']]
        for n, c0, c1 in _chunks(s):
            if k == 'up':
                raw = s['x'][n, ..., c0:c1].permute(2, 0, 1).double()[None]
                acc = oo.upfirdn2d(raw, f64, padding=1, gain=4)[0].permute(1, 2, 0)
                del raw
            else:
                acc = s['x'][:, n, ..., c0:c1].double().sum(0)
            v = epilogue_reference(acc, s, n, c0, c1)
            if s['f32'] is not None:
                co = c['f32']['coff']
                e_f32.add(s['f32'].view[n, ..., co + c0:co + c1], v)
            for e, (hi, lo, sty), o in zip(e_split, s['outs'], c['outs']):
                ref = v * sty[n, c0:c1].double() if sty is not None else v
                co = o['coff']
                e.add(hi.view[n, ..., co + c0:co + c1].double() + lo.view[n, ..., co + c0:co + c1].double(), ref)
            del acc, v
        if s['f32'] is not None:
            errs[f'{k}.f32'] = e_f32.value()
        if e_split:
            errs[f'{k}.split'] = max(e.value() for e in e_split)
    elif k == 'modsplit':
        e = RangeErr()
        (hi, lo, sty), o = s['outs'][0], c['outs'][0]
        for n, c0, c1 in _chunks(s):
            ref = s['x'][n, ..., c0:c1].double() * (sty[n, c0:c1].double() if sty is not None else 1.0)
            co = o['coff']
            e.add(hi.view[n, ..., co + c0:co + c1].double() + lo.view[n, ..., co + c0:co + c1].double(), ref)
        errs['modsplit.split'] = e.value()
    elif k == 'down':
        e = RangeErr()
        hi, lo, _ = s['outs'][0]
        H, W = c['H'], c['W']
        SH, SW = (H + 2) // 2, (W + 2) // 2
        # the pad row and column beyond the (H+1) x (W+1) FIR output are exact zeros (parities with a = 1 / b = 1)
        for t in (hi, lo):
            bits = t.bits()
            assert (bits[2:, :, SH - 1] == 0).all() and (bits[1::2, :, :, SW - 1] == 0).all(), f'{c["name"]}: pad row / column not zero'
        for n, c0, c1 in _chunks(s):
            x = s['x'][n, ..., c0:c1].permute(2, 0, 1).double()[None]
            fo = F.pad(oo.upfirdn2d(x, f64, padding=2)[0], (0, 1, 0, 1))       # (H+2) x (W+2): the extra row / column is the zero pad
            for a in (0, 1):
                for b in (0, 1):
                    p = a * 2 + b
                    e.add(hi.view[p, n, ..., c0:c1].double() + lo.view[p, n, ..., c0:c1].double(), fo[:, a::2, b::2].permute(1, 2, 0))
            del x, fo
        errs['down.split'] = e.value()
    else:
        e = RangeErr()
        fn = oo.upsample2d if k == 'upsample' else oo.downsample2d
        for n, c0, c1 in _chunks(s):
            ref = fn(s['x'][n, ..., c0:c1].permute(2, 0, 1).double()[None], f64)[0]
            got = s['f32'].view[n, c0:c1] if c['nchw'] else s['f32'].view[n, ..., c0:c1].permute(2, 0, 1)
            e.add(got, ref)
        errs[k] = e.value()
    return errs


@pytest.mark.gpu
@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_kernel_matches_fp64_reference(c, monkeypatch):
    monkeypatch.delenv('N3D_FIR_STREAM', raising=False)
    s = setup_case(c)
    launch_case(s)
    torch.cuda.synchronize()
    errs = check_case(s)
    record_errors('N3D_FIR_ERRORS', [{'case': c['name'], 'kind': k, 'err': e, 'bound': BOUNDS[k]} for k, e in errs.items()])
    bad = {k: e for k, e in errs.items() if not e < BOUNDS[k]}
    assert not bad, bad
    rerun = lambda: rerun_identical(outputs(s), lambda: launch_case(s))        # noqa: E731
    assert rerun(), f'{c["name"]}: a rerun is not bit-identical'
    if plan(c, torch.cuda.get_device_properties(0).multi_processor_count)['streamed']:
        monkeypatch.setenv('N3D_FIR_STREAM', '0')
        assert rerun(), f'{c["name"]}: the register-tiled kernel is not bit-identical to the streamed one'


@pytest.mark.gpu
def test_launched_kernel_matches_plan(tmp_path, monkeypatch):
    """Every case under torch.profiler: the kernel it launched and its grid are the ones `plan` predicts at the device's SM count."""
    monkeypatch.delenv('N3D_FIR_STREAM', raising=False)
    pattern = re.compile(r'fir_up_stream_kernel|fir_up_epilogue_kernel|fir_down_stream_kernel|fir_down_split_kernel|upsample2d_kernel<\d>|'
                         r'downsample2d_kernel|modulate_split_kernel|splitk_epilogue_kernel')

    def run():
        for c in CASES:                     # one case at a time: the largest ones do not fit in memory together
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


# ------------------------------------------------------------------------------------------------ alignment (CPU, nothing launched)
@pytest.mark.parametrize('field', ['x', 'hi', 'lo'])
def test_fir_down_split_refuses_misaligned_pointers(field):
    L = lib()
    N, H, W, Cc = 1, 8, 8, 16
    x = torch.zeros(N * H * W * Cc + 64)
    bf = {k: torch.zeros(4 * N * 5 * 5 * Cc + 64, dtype=torch.bfloat16) for k in ('hi', 'lo')}
    p = dict(x=x.data_ptr(), hi=bf['hi'].data_ptr(), lo=bf['lo'].data_ptr())
    p[field] = offset_view(x if field == 'x' else bf[field], 4).data_ptr()
    what = 'x must be 16-byte aligned' if field == 'x' else 'hi and lo must be 8-byte aligned'
    refused(L.lib.n3d_fir_down_split(p['x'], N, H, W, Cc, p['hi'], p['lo'], None), what)


@pytest.mark.parametrize('field', ['x', 'style', 'hi', 'lo'])
def test_modulate_split_refuses_misaligned_pointers(field):
    L = lib()
    N, HW, Cc = 1, 16, 16
    f32 = {k: torch.zeros(N * HW * Cc + 64) for k in ('x', 'style')}
    bf = {k: torch.zeros(N * HW * Cc + 64, dtype=torch.bfloat16) for k in ('hi', 'lo')}
    t = {**f32, **bf}
    p = {k: v.data_ptr() for k, v in t.items()}
    p[field] = offset_view(t[field], 4).data_ptr()
    what = 'x and style must be 16-byte aligned' if field in f32 else 'hi and lo must be 8-byte aligned'
    refused(L.lib.n3d_modulate_split(p['x'], HW, N, Cc, p['style'], p['hi'], p['lo'], Cc, 0, None), what)


@pytest.mark.parametrize('field', ['blended_front', 'tex_planes', 'static_planes', 'planes'])
def test_blend_planes_refuses_misaligned_pointers(field):
    L = lib()
    N, H, W = 1, 4, 4
    t = dict(blended_front=torch.zeros(N * H * W * 32 + 64), tex_planes=torch.zeros(3 * N * H * W * 32 + 64),
             static_planes=torch.zeros(N * H * W * 96 + 64), planes=torch.zeros(N * 3 * H * W * 32 + 64))
    alpha = torch.zeros(3 * N * H * W)
    p = {k: v.data_ptr() for k, v in t.items()}
    p[field] = offset_view(t[field], 4).data_ptr()
    refused(L.lib.n3d_blend_planes(p['blended_front'], p['tex_planes'], alpha.data_ptr(), p['static_planes'], N, H, W, p['planes'], None),
             'blended_front, tex_planes, static_planes and planes must be 16-byte aligned')


@pytest.mark.gpu
@pytest.mark.parametrize('nchw', [False, True])
def test_upsample2d_takes_scalar_path_for_misaligned_pointers(nchw):
    """n3d_upsample2d_nhwc at C % 4 == 0 with x (and y) starting 4 bytes into their allocation: one channel per thread, same result."""
    from next3d_b200 import kernels as K
    from oracle import ops as oo
    N, H, W, Cc = 2, 5, 7, 8
    x = offset_view(torch.randn(N * H * W * Cc + 64, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7)), 4)[:N * H * W * Cc]
    y = offset_view(torch.full((N * 4 * H * W * Cc + 64,), float('nan'), device=DEV), 4)[:N * 4 * H * W * Cc]
    y = y.view(N, Cc, 2 * H, 2 * W) if nchw else y.view(N, 2 * H, 2 * W, Cc)
    K.upsample2d_nhwc(x.view(N, H, W, Cc), y, y_nchw=nchw)
    ref = oo.upsample2d(x.view(N, H, W, Cc).permute(0, 3, 1, 2).double(), _filter64())
    got = y if nchw else y.permute(0, 3, 1, 2)
    err = ((got.double() - ref).abs().max() / ref.abs().max()).item()
    record_errors('N3D_FIR_ERRORS', [{'case': f'upsample_misaligned_{"nchw" if nchw else "nhwc"}', 'kind': 'upsample', 'err': err,
                                      'bound': BOUNDS['upsample']}])
    assert err < BOUNDS['upsample'], err
