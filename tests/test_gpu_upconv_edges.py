"""n3d_conv_transposed_gemm runs the four output-parity classes of a stride-2 transposed 3x3 conv in one launch: the H x W interior
of every class as interleaved sub-problems, and the extra row / column / corner of the (H+1)-sized classes as thin edge
sub-problems with tile shapes of their own.  Every output pixel must see the same taps in the same order as when its class runs
as a separate n3d_conv_gemm launch, so the raw output must match the four-launch result bit for bit, with every pixel written."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.helpers import range_rel_err

pytestmark = pytest.mark.gpu

DEV = 'cuda'


@pytest.fixture(scope='module')
def K():
    from next3d_b200 import kernels
    return kernels


def _run_both(K, N, Cin, Cout, res, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, res, res, Cin, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(Cin * 9)
    a_hi, a_lo = K.split_bf16(x.to(DEV))
    w_hi, w_lo = K.pack_conv_weight(w.to(DEV))
    raw4 = torch.full((N, 2 * res + 1, 2 * res + 1, Cout), float('nan'), device=DEV)
    for a in (0, 1):
        for b in (0, 1):
            K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_transposed(a, b), N, res + 1 - a, res + 1 - b, mode=1, out_f32=raw4,
                        f32_cstride=Cout, oy_mul=2, oy_off=a, ox_mul=2, ox_off=b, OH=2 * res + 1, OW=2 * res + 1)
    raw1 = torch.full_like(raw4, float('nan'))
    K.conv_transposed_gemm(a_hi, a_lo, w_hi, w_lo, N, res, res, raw1)
    torch.cuda.synchronize()
    return x, w, a_hi, a_lo, raw4, raw1


# TN > 1 interiors (4^2: 4x4x8 tiles, 8^2: 8x8x2), N not a multiple of TN, several n-tiles (Cout 256 / 512), odd and
# non-power-of-two sizes, and enough tiles for the grouped work order (more parity-class items than SMs).
@pytest.mark.parametrize('N,Cin,Cout,res', [(8, 64, 64, 4), (3, 64, 64, 4), (5, 32, 96, 8), (2, 64, 256, 16), (1, 64, 512, 8),
                                            (3, 32, 64, 37), (2, 64, 128, 64), (1, 128, 256, 96)])
def test_transposed_one_launch_matches_four(K, N, Cin, Cout, res):
    x, w, a_hi, a_lo, raw4, raw1 = _run_both(K, N, Cin, Cout, res, 41 + N + Cin + Cout + res)
    assert not torch.isnan(raw1).any()
    assert torch.equal(raw4, raw1)
    # the raw result is conv_transpose2d(stride 2) of the split-rounded input (fp32 = hi + lo)
    xs = (a_hi.float() + a_lo.float()).cpu().permute(0, 3, 1, 2).double()
    ref = F.conv_transpose2d(xs, w.double().permute(1, 0, 2, 3), stride=2).float()
    assert range_rel_err(raw1.permute(0, 3, 1, 2).cpu(), ref) < 3e-5


def test_transposed_c2_shape_bit_identical(K):
    """b256.conv0 at c2: input 128^2, Cin 256 -> Cout 128, batch 8."""
    *_, raw4, raw1 = _run_both(K, 8, 256, 128, 128, 5)
    assert not torch.isnan(raw1).any()
    assert torch.equal(raw4, raw1)
