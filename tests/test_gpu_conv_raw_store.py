"""The raw fp32 output of conv_gemm (mode 1: transposed convolutions, split-K partial sums) against the fp64 contract, at shapes
where the TMA store boxes hang over what a launch owns: M-spaces that are not whole tiles, N not a multiple of TN, Cout tails
inside a box, a channel window (f32_coff, f32_cstride > Cout) of a wider buffer, cluster pad tiles, split-K slices, M rows that
fall outside OH, transposed launches at small odd sizes, and a descriptor the TMA cannot express (per-thread stores).

Every output is a view into a NaN-sentinel allocation (tests/helpers.Guarded): the owned elements must be written and match the
reference within the conformance suite's bound for raw output; every other element must keep the sentinel's bits."""
import math

import pytest
import torch

from tests.helpers import Guarded
from tests.test_gpu_conv_conformance import BOUNDS, conv_reference, plan

pytestmark = pytest.mark.gpu

DEV = 'cuda'

# name, N, Cin, Cout, MH x MW M-space; optional: splits (K slices), cstride / coff (f32_cstride / f32_coff), cls = (a, b): the
# M-space is parity class (a, b) of a stride-2 transposed conv of an (MH - 1) x (MW - 1) input, and its last row / column falls
# outside OH / OW unless a / b is 0
CASES = [
    dict(name='mspace_tails_cout_tail', N=3, Cin=48, Cout=40, MH=11, MW=21),
    dict(name='tn8_n_tail', N=5, Cin=32, Cout=64, MH=4, MW=4),
    dict(name='tn2_n_tail', N=3, Cin=64, Cout=32, MH=8, MW=8),
    dict(name='channel_window', N=2, Cin=40, Cout=24, MH=9, MW=17, cstride=40, coff=8),
    dict(name='bn16_swizzle64', N=2, Cin=24, Cout=12, MH=16, MW=13, cstride=16, coff=4),
    dict(name='bn128_cluster_pad', N=33, Cin=8, Cout=256, MH=8, MW=16),
    dict(name='bn96_cluster_pad', N=65, Cin=16, Cout=96, MH=8, MW=16),
    dict(name='splitk9', N=2, Cin=64, Cout=64, MH=4, MW=4, splits=9),
    dict(name='splitk3_tails', N=3, Cin=80, Cout=40, MH=5, MW=7, splits=3),
    dict(name='splitk2_uneven', N=2, Cin=24, Cout=72, MH=8, MW=8, splits=2),
    dict(name='class11_rows_past_oh', N=2, Cin=32, Cout=48, MH=6, MW=8, cls=(1, 1)),
    dict(name='class00_strided', N=3, Cin=16, Cout=32, MH=6, MW=5, cls=(0, 0), cstride=36, coff=4),
    dict(name='fallback_cstride41', N=2, Cin=32, Cout=40, MH=7, MW=9, cstride=41, coff=1),
]
TRANSPOSED = [(2, 40, 48, 3, 5), (3, 32, 128, 7, 7), (1, 16, 64, 1, 1), (5, 24, 96, 5, 3)]     # N, Cin, Cout, H, W


def _operands(N, Cin, Cout, H, W, T, ntaps, seed):
    from next3d_b200 import kernels as K
    g = torch.Generator(device=DEV).manual_seed(seed)
    a_hi, a_lo = K.split_bf16(torch.randn(N, H, W, Cin, device=DEV, generator=g))
    w_hi, w_lo = K.split_bf16(torch.randn(T, Cout, Cin, device=DEV, generator=g) / math.sqrt(Cin * ntaps))
    return a_hi, a_lo, w_hi, w_lo


def _check(out, expect):
    assert out.untouched_ok(), 'an element outside the output was written'
    assert out.written(), 'an owned element was not written'
    got, ref = out.view[out.own].double(), expect[out.own]
    err = ((got - ref).abs().max() / ref.abs().max()).item()
    assert err < BOUNDS['raw'], err


@pytest.mark.parametrize('c', CASES, ids=[c['name'] for c in CASES])
def test_raw_output_matches_fp64_contract(c):
    from next3d_b200 import kernels as K
    N, Cin, Cout, MH, MW = c['N'], c['Cin'], c['Cout'], c['MH'], c['MW']
    S, cs, coff = c.get('splits', 1), c.get('cstride', Cout), c.get('coff', 0)
    if 'cls' in c:                          # parity class (a, b) of a transposed conv of an (MH - 1) x (MW - 1) input
        a, b = c['cls']
        H, W = MH - 1, MW - 1
        taps, oy_mul, ox_mul, oy_off, ox_off, OH, OW = K.taps_transposed(a, b), 2, 2, a, b, 2 * H + 1, 2 * W + 1
    else:
        H, W = MH, MW
        taps, oy_mul, ox_mul, oy_off, ox_off, OH, OW = K.taps_conv3x3(), 1, 1, 0, 0, MH, MW
    a_hi, a_lo, w_hi, w_lo = _operands(N, Cin, Cout, H, W, 9, len(taps), 7 + sum(map(ord, c['name'])))
    out = Guarded(((S,) if S > 1 else ()) + (N, OH, OW, cs), own=torch.zeros(((S,) if S > 1 else ()) + (N, OH, OW, cs), dtype=torch.bool, device=DEV))
    K.conv_gemm(a_hi, a_lo, w_hi, w_lo, taps, N, MH, MW, mode=1, out_f32=out.view, f32_cstride=cs, f32_coff=coff, oy_mul=oy_mul,
                oy_off=oy_off, ox_mul=ox_mul, ox_off=ox_off, OH=OH, OW=OW, splits=S, split_stride=out.view[0].numel() if S > 1 else 0)
    torch.cuda.synchronize()
    # owned: M pixels whose output position lies inside OH x OW, channels [coff, coff + Cout), every K slice
    ys = torch.arange(MH, device=DEV) * oy_mul + oy_off
    xs = torch.arange(MW, device=DEV) * ox_mul + ox_off
    yv, xv = torch.nonzero(ys < OH).flatten(), torch.nonzero(xs < OW).flatten()
    expect = torch.zeros(out.view.shape, dtype=torch.float64, device=DEV)
    block_k = plan(N, Cin, Cout, MH, MW, S)['block_k']
    per = -(-len(taps) * -(-Cin // block_k) // S)          # K steps per slice (k_range in conv_gemm.cu)
    n = torch.arange(N, device=DEV)[:, None, None, None]
    ch = torch.arange(Cout, device=DEV)[None, None, None, :] + coff
    Y, X = ys[yv][None, :, None, None], xs[xv][None, None, :, None]
    for k in range(S):
        kw = dict(block_k=block_k, k_steps=(k * per, (k + 1) * per)) if S > 1 else {}
        acc = conv_reference(a_hi, a_lo, w_hi, w_lo, taps, N, MH, MW, **kw)[:, yv][:, :, xv]
        idx = ((torch.full_like(n, k),) if S > 1 else ()) + (n, Y, X, ch)
        out.own[idx] = True
        expect[idx] = acc
    _check(out, expect)


@pytest.mark.parametrize('N,Cin,Cout,H,W', TRANSPOSED)
def test_transposed_raw_output_matches_fp64_contract(N, Cin, Cout, H, W):
    from next3d_b200 import kernels as K
    a_hi, a_lo, w_hi, w_lo = _operands(N, Cin, Cout, H, W, 9, 4, 11 + N + Cin + Cout + H * W)
    OH, OW = 2 * H + 1, 2 * W + 1
    out = Guarded((N, OH, OW, Cout))
    K.conv_transposed_gemm(a_hi, a_lo, w_hi, w_lo, N, H, W, out.view)
    torch.cuda.synchronize()
    expect = torch.zeros(out.view.shape, dtype=torch.float64, device=DEV)
    for a in (0, 1):
        for b in (0, 1):
            expect[:, a::2, b::2] = conv_reference(a_hi, a_lo, w_hi, w_lo, K.taps_transposed(a, b), N, H + 1 - a, W + 1 - b)
    out.own = torch.ones(out.view.shape, dtype=torch.bool, device=DEV)
    _check(out, expect)
