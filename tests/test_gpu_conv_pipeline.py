"""conv_gemm work items that span several n-tiles: the fused ToRGB at Cout 256 runs each 128-pixel tile as two 128-wide n-tiles in
turn, carrying the ToRGB partial sums across them.  The cases reuse the reference check of tests/test_gpu_kernels.py; the larger
ones give every CTA several work items, so both ping-pong warpgroups take items and step their ring positions past each other's."""
import math

import pytest
import torch

from tests.test_gpu_kernels import test_conv_fused_torgb as check_fused_torgb

pytestmark = pytest.mark.gpu

DEV = 'cuda'


@pytest.fixture(scope='module')
def K():
    from next3d_b200 import kernels
    return kernels


# work items = N * res^2 / 128 (one per 128-pixel tile): 64 (fewer than the SMs: one item per CTA), 1024 and 128
@pytest.mark.parametrize('N,Cin,Cout,res,nchw,with_out', [(2, 256, 256, 64, True, True), (2, 64, 256, 256, False, True),
                                                         (1, 32, 256, 128, True, False)])
def test_conv_fused_torgb_multi_ntile(K, N, Cin, Cout, res, nchw, with_out):
    check_fused_torgb(K, N, Cin, Cout, res, nchw, with_out)


@pytest.mark.parametrize('Cin,Cout,res', [(64, 256, 256), (128, 128, 128)])
def test_conv_fused_torgb_bit_reproducible(K, Cin, Cout, res):
    """Fixed summation order (no atomics): two launches give the same image bit for bit."""
    g = torch.Generator(device=DEV).manual_seed(29 + Cout)
    N = 2
    a_hi, a_lo = K.split_bf16(torch.randn(N, res, res, Cin, device=DEV, generator=g))
    w_hi, w_lo = K.pack_conv_weight(torch.randn(Cout, Cin, 3, 3, device=DEV, generator=g) / math.sqrt(Cin * 9))
    # descriptors hold raw device pointers: every operand stays referenced for the whole test
    d = torch.rand(N, Cout, device=DEV, generator=g) + 0.5
    b = torch.randn(Cout, device=DEV, generator=g)
    sr = torch.randn(N, Cout, device=DEV, generator=g) / math.sqrt(Cout)
    wr = torch.randn(3, Cout, device=DEV, generator=g)
    br = torch.randn(3, device=DEV, generator=g)
    prev = torch.randn(N, 3, res, res, device=DEV, generator=g)

    def run():
        img = prev.clone()
        K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_conv3x3(), N, res, res, dcoef=d, bias=b, gain=math.sqrt(2), slope=0.2, clamp=256.0,
                    outs=[], rgb=dict(out=img, weight=wr, style=sr, bias=br, clamp=2.0, nchw=True, accumulate=True))
        return img

    first = run()
    assert torch.equal(run(), first)
