"""conv_gemm launches as 2-CTA clusters that share the weight tile.  A launch of N images of 16x8 pixels has one 128-pixel M tile
per image, so with block_n >= 96 the M tiles are paired across a cluster, and an odd N leaves a pad tile.  The same images run as
N one-image launches have a single M tile each and stay unclustered.  Which CTA computes a tile does not change its (tap,
16-channel, product) accumulation order, so both must agree bit for bit."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = 'cuda'
H, W = 8, 16                       # one 16 x 8 tile per image


@pytest.fixture(scope='module')
def K():
    from next3d_b200 import kernels
    return kernels


def _operands(K, N, Cin, Cout, seed, h=H, w=W):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a_hi, a_lo = K.split_bf16(torch.randn(N, h, w, Cin, device=DEV, generator=g))
    w_hi, w_lo = K.pack_conv_weight(torch.randn(Cout, Cin, 3, 3, device=DEV, generator=g) / math.sqrt(Cin * 9))
    return g, a_hi, a_lo, w_hi, w_lo


# N * tiles_n >= 64 keeps block_n at 128 (96 for Cout 96); odd N: the last cluster pairs a tile with a pad tile
@pytest.mark.parametrize('N,Cin,Cout', [(33, 64, 256), (65, 96, 96), (33, 128, 200), (64, 64, 128)])
def test_clustered_conv_matches_one_image_launches(K, N, Cin, Cout):
    g, a_hi, a_lo, w_hi, w_lo = _operands(K, N, Cin, Cout, 11 + N + Cout)
    bias = torch.randn(Cout, device=DEV, generator=g)
    dcoef = torch.rand(N, Cout, device=DEV, generator=g) + 0.5
    raw = torch.full((N, H, W, Cout), float('nan'), device=DEV)
    K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_conv3x3(), N, H, W, mode=1, dcoef=dcoef, bias=bias, out_f32=raw, f32_cstride=Cout)
    ref = torch.full_like(raw, float('nan'))
    for n in range(N):
        K.conv_gemm(a_hi[n:n + 1], a_lo[n:n + 1], w_hi, w_lo, K.taps_conv3x3(), 1, H, W, mode=1, dcoef=dcoef[n:n + 1], bias=bias,
                    out_f32=ref[n:n + 1], f32_cstride=Cout)
    torch.cuda.synchronize()
    assert torch.equal(raw, ref)


def test_clustered_fused_torgb_matches_one_image_launches(K):
    """Cout 256: each work item runs two 128-wide n-tiles in turn; the pad tile of N = 33 must write no ToRGB pixel."""
    N, Cin, Cout = 33, 64, 256
    g, a_hi, a_lo, w_hi, w_lo = _operands(K, N, Cin, Cout, 5)
    d = torch.rand(N, Cout, device=DEV, generator=g) + 0.5
    b = torch.randn(Cout, device=DEV, generator=g)
    sr = torch.randn(N, Cout, device=DEV, generator=g) / math.sqrt(Cout)
    wr = torch.randn(3, Cout, device=DEV, generator=g)
    br = torch.randn(3, device=DEV, generator=g)
    prev = torch.randn(N, 3, H, W, device=DEV, generator=g)

    def run(n0, n1, img):
        K.conv_gemm(a_hi[n0:n1], a_lo[n0:n1], w_hi, w_lo, K.taps_conv3x3(), n1 - n0, H, W, dcoef=d[n0:n1], bias=b, gain=math.sqrt(2),
                    slope=0.2, clamp=256.0, outs=[],
                    rgb=dict(out=img, weight=wr, style=sr[n0:n1], bias=br, clamp=2.0, nchw=True, accumulate=True))

    img = prev.clone()
    run(0, N, img)
    ref = prev.clone()
    for n in range(N):
        run(n, n + 1, ref[n:n + 1])
    torch.cuda.synchronize()
    assert torch.equal(img, ref)


def test_clustered_transposed_conv_matches_one_image_launches(K):
    """Nine sub-problems (four parity-class interiors, two row strips, two column strips, the corner pixel); N = 9 gives the
    interiors an odd tile count and the strips and the corner a single M tile each, paired with a pad tile."""
    N, Cin, Cout = 9, 64, 256
    _, a_hi, a_lo, w_hi, w_lo = _operands(K, N, Cin, Cout, 3)
    raw = torch.full((N, 2 * H + 1, 2 * W + 1, Cout), float('nan'), device=DEV)
    K.conv_transposed_gemm(a_hi, a_lo, w_hi, w_lo, N, H, W, raw)
    ref = torch.full_like(raw, float('nan'))
    for n in range(N):
        K.conv_transposed_gemm(a_hi[n:n + 1], a_lo[n:n + 1], w_hi, w_lo, 1, H, W, ref[n:n + 1])
    torch.cuda.synchronize()
    assert torch.equal(raw, ref)


def test_clustered_conv_graph_replay_matches_eager(K):
    N, Cin, Cout = 33, 64, 256
    _, a_hi, a_lo, w_hi, w_lo = _operands(K, N, Cin, Cout, 7)
    eager = torch.empty(N, H, W, Cout, device=DEV)
    K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_conv3x3(), N, H, W, mode=1, out_f32=eager, f32_cstride=Cout)
    out = torch.full_like(eager, float('nan'))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_conv3x3(), N, H, W, mode=1, out_f32=out, f32_cstride=Cout)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
