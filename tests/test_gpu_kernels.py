"""GPU parity tests, kernel by kernel, through the C ABI (ctypes) against the CPU oracle.

Tolerances (range-relative, max|d|/max|ref|): tensor-core convolutions use the 3-product bf16 split scheme, i.e.
~2^-16 per product -> 3e-5; fp32 SIMT kernels 1e-5; the rasterizer index buffer must be bit-exact.
"""
import math

import numpy as np
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


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _nhwc_split(K, x_nchw):
    x = x_nchw.permute(0, 2, 3, 1).contiguous().to(DEV)
    return K.split_bf16(x)


def _join(hi, lo):
    return hi.float() + lo.float()


# ------------------------------------------------------------------------------------------------ conv_gemm
@pytest.mark.parametrize('N,Cin,Cout,res', [(1, 32, 32, 16), (2, 64, 128, 16), (8, 512, 512, 4), (2, 512, 512, 8), (1, 128, 96, 32),
                                           (1, 256, 3, 32), (2, 16, 16, 64), (1, 128, 256, 64), (3, 96, 64, 24), (1, 1024, 512, 8),
                                           (1, 32, 256, 128),
                                           (2, 32, 128, 280), (1, 64, 128, 400)])      # block_n 128, >= 8 waves of tiles
def test_conv3x3_plain(K, N, Cin, Cout, res):
    g = _g(N * 1000 + Cin + Cout + res)
    x = torch.randn(N, Cin, res, res, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(Cin * 9)
    ref = F.conv2d(x.double(), w.double(), padding=1).float()
    a_hi, a_lo = _nhwc_split(K, x)
    w_hi, w_lo = K.pack_conv_weight(w.to(DEV))
    out = torch.full((N, res, res, Cout), float('nan'), device=DEV)
    K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_conv3x3(), N, res, res, out_f32=out, f32_cstride=Cout)
    torch.cuda.synchronize()
    got = out.permute(0, 3, 1, 2).cpu()
    assert range_rel_err(got, ref) < 6e-5


def test_conv_single_product_is_bf16_grade(K):
    g = _g(7)
    x = torch.randn(1, 64, 16, 16, generator=g)
    w = torch.randn(64, 64, 3, 3, generator=g) / 24
    ref = F.conv2d(x.double(), w.double(), padding=1).float()
    a_hi, a_lo = _nhwc_split(K, x)
    w_hi, w_lo = K.pack_conv_weight(w.to(DEV))
    out = torch.zeros(1, 16, 16, 64, device=DEV)
    K.conv_gemm(a_hi, None, w_hi, None, K.taps_conv3x3(), 1, 16, 16, nprod=1, out_f32=out, f32_cstride=64)
    err = range_rel_err(out.permute(0, 3, 1, 2).cpu(), ref)
    assert 1e-4 < err < 2e-2      # bf16 x bf16 single product: clearly worse than the split scheme, clearly a conv


def test_conv_epilogue_full(K):
    """demod + noise + bias + lrelu*sqrt2 + clamp, two modulated split outputs into a concat buffer, fp32 copy."""
    g = _g(11)
    N, Cin, Cout, res = 2, 64, 128, 32
    x = torch.randn(N, Cin, res, res, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(Cin * 9)
    d = torch.rand(N, Cout, generator=g) + 0.5
    b = torch.randn(Cout, generator=g)
    nz = torch.randn(res, res, generator=g) * 0.1
    s1 = torch.randn(N, Cout, generator=g)
    s2 = torch.randn(N, Cout, generator=g)
    y = F.conv2d(x, w, padding=1) * d[:, :, None, None] + nz[None, None]
    y = (F.leaky_relu(y + b[None, :, None, None], 0.2) * math.sqrt(2)).clamp(-1.5, 1.5)
    a_hi, a_lo = _nhwc_split(K, x)
    w_hi, w_lo = K.pack_conv_weight(w.to(DEV))
    cat_hi = torch.zeros(N, res, res, 2 * Cout, device=DEV, dtype=torch.bfloat16)
    cat_lo = torch.zeros_like(cat_hi)
    o2_hi = torch.zeros(N, res, res, Cout, device=DEV, dtype=torch.bfloat16)
    o2_lo = torch.zeros_like(o2_hi)
    f32 = torch.zeros(N, res, res, Cout, device=DEV)
    dd, bd, nzd, s1d, s2d = d.to(DEV), b.to(DEV), nz.to(DEV), s1.to(DEV), s2.to(DEV)    # keep the device tensors alive: raw pointers are passed
    K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_conv3x3(), N, res, res, dcoef=dd, bias=bd, noise=nzd,
                gain=math.sqrt(2), slope=0.2, clamp=1.5,
                outs=[K.make_split_out(cat_hi, cat_lo, s1d, 2 * Cout, Cout), K.make_split_out(o2_hi, o2_lo, s2d, Cout, 0)],
                out_f32=f32, f32_cstride=Cout)
    assert range_rel_err(f32.permute(0, 3, 1, 2).cpu(), y) < 3e-5
    assert range_rel_err(_join(cat_hi, cat_lo)[..., Cout:].permute(0, 3, 1, 2).cpu(), y * s1[:, :, None, None]) < 5e-5
    assert _join(cat_hi, cat_lo)[..., :Cout].abs().max().item() == 0.0      # left half of the concat buffer untouched
    assert range_rel_err(_join(o2_hi, o2_lo).permute(0, 3, 1, 2).cpu(), y * s2[:, :, None, None]) < 5e-5


def test_conv1x1_torgb_nchw_accumulate(K):
    g = _g(13)
    N, Cin, res = 2, 128, 32
    x = torch.randn(N, Cin, res, res, generator=g)
    w = torch.randn(3, Cin, 1, 1, generator=g) / math.sqrt(Cin)
    b = torch.randn(3, generator=g)
    prev = torch.randn(N, 3, res, res, generator=g)
    ref = prev + (F.conv2d(x, w) + b[None, :, None, None]).clamp(-256, 256)
    a_hi, a_lo = _nhwc_split(K, x)
    w_hi, w_lo = K.pack_conv_weight(w.to(DEV))
    out = prev.clone().to(DEV)
    K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_conv1x1(), N, res, res, bias=b.to(DEV), clamp=256.0, out_f32=out, f32_cstride=3,
                f32_nchw=True, f32_accumulate=True)
    assert range_rel_err(out.cpu(), ref) < 3e-5


@pytest.mark.parametrize('per_sample_noise', [False, True], ids=['shared-noise', 'per-sample-noise'])
@pytest.mark.parametrize('N,Cin,Cout,res,S', [(8, 512, 512, 4, 9), (8, 512, 512, 8, 9), (2, 32, 32, 16, 9), (3, 1024, 512, 8, 4), (1, 64, 96, 8, 3)])
def test_conv_splitk(K, N, Cin, Cout, res, S, per_sample_noise):
    """Split-K (deterministic two-pass): S K-slices write raw partial sums, n3d_splitk_epilogue sums them in fixed order and applies
    the SynthesisLayer epilogue.  Same result as the one-pass kernel (up to fp32 summation order) and bit-reproducible.  Noise is one
    map for the batch ('const') or one per image (noise_nstride = H * W, 'random')."""
    g = _g(23 + Cin + res)
    x = torch.randn(N, Cin, res, res, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(Cin * 9)
    d = torch.rand(N, Cout, generator=g) + 0.5
    b = torch.randn(Cout, generator=g)
    nz = torch.randn(*((N,) if per_sample_noise else ()), res, res, generator=g) * 0.1
    nstride = res * res if per_sample_noise else 0
    s1 = torch.randn(N, Cout, generator=g)
    y = F.conv2d(x.double(), w.double(), padding=1).float() * d[:, :, None, None] + nz.reshape(-1, 1, res, res)
    y = (F.leaky_relu(y + b[None, :, None, None], 0.2) * math.sqrt(2)).clamp(-2.0, 2.0)
    a_hi, a_lo = _nhwc_split(K, x)
    w_hi, w_lo = K.pack_conv_weight(w.to(DEV))
    dd, bd, nzd, s1d = d.to(DEV), b.to(DEV), nz.to(DEV), s1.to(DEV)

    def run():
        part = torch.full((S, N, res, res, Cout), float('nan'), device=DEV)
        K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_conv3x3(), N, res, res, mode=1, out_f32=part, f32_cstride=Cout, splits=S,
                    split_stride=N * res * res * Cout)
        assert not torch.isnan(part).any()
        o_hi = torch.zeros(N, res, res, Cout, device=DEV, dtype=torch.bfloat16)
        o_lo = torch.zeros_like(o_hi)
        f32 = torch.zeros(N, res, res, Cout, device=DEV)
        K.splitk_epilogue(part, dd, bd, nzd, math.sqrt(2), 0.2, 2.0, outs=[K.make_split_out(o_hi, o_lo, s1d, Cout, 0)], out_f32=f32, f32_cstride=Cout,
                          noise_nstride=nstride)
        return f32, o_hi, o_lo

    f32, o_hi, o_lo = run()
    assert range_rel_err(f32.permute(0, 3, 1, 2).cpu(), y) < 6e-5
    assert range_rel_err(_join(o_hi, o_lo).permute(0, 3, 1, 2).cpu(), y * s1[:, :, None, None]) < 8e-5
    f32b, _, _ = run()
    assert torch.equal(f32, f32b)


@pytest.mark.parametrize('N,Cin,Cout,res,nchw,with_out', [(2, 64, 128, 32, True, True), (1, 128, 256, 16, False, True), (2, 32, 128, 32, True, False),
                                                         (2, 32, 128, 280, True, False)])     # last: block_n 128, >= 8 waves of tiles
def test_conv_fused_torgb(K, N, Cin, Cout, res, nchw, with_out):
    """ToRGBLayer (networks_stylegan2.py:353-357) folded into the producing conv's epilogue: img += clamp(W_rgb (y * s_rgb) + b_rgb),
    optionally with no other output of the conv at all (last super-resolution layer)."""
    g = _g(19 + Cout + res)
    x = torch.randn(N, Cin, res, res, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(Cin * 9)
    d = torch.rand(N, Cout, generator=g) + 0.5
    b = torch.randn(Cout, generator=g)
    s_next = torch.randn(N, Cout, generator=g)
    s_rgb = torch.randn(N, Cout, generator=g) / math.sqrt(Cout)
    w_rgb = torch.randn(3, Cout, generator=g)
    b_rgb = torch.randn(3, generator=g)
    prev = torch.randn(N, 3, res, res, generator=g)
    y = (F.leaky_relu(F.conv2d(x, w, padding=1) * d[:, :, None, None] + b[None, :, None, None], 0.2) * math.sqrt(2)).clamp(-256, 256)
    rgb = torch.einsum('nchw,nc,kc->nkhw', y.double(), s_rgb.double(), w_rgb.double()).float() + b_rgb[None, :, None, None]
    ref = prev + rgb.clamp(-2.0, 2.0)
    a_hi, a_lo = _nhwc_split(K, x)
    w_hi, w_lo = K.pack_conv_weight(w.to(DEV))
    img = (prev if nchw else prev.permute(0, 2, 3, 1)).contiguous().to(DEV)
    o_hi = torch.zeros(N, res, res, Cout, device=DEV, dtype=torch.bfloat16)
    o_lo = torch.zeros_like(o_hi)
    dd, bd, sn, sr, wr, br = d.to(DEV), b.to(DEV), s_next.to(DEV), s_rgb.to(DEV), w_rgb.to(DEV), b_rgb.to(DEV)
    K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_conv3x3(), N, res, res, dcoef=dd, bias=bd, gain=math.sqrt(2), slope=0.2, clamp=256.0,
                outs=[K.make_split_out(o_hi, o_lo, sn, Cout, 0)] if with_out else [],
                rgb=dict(out=img, weight=wr, style=sr, bias=br, clamp=2.0, nchw=nchw, accumulate=True))
    got = img.cpu() if nchw else img.permute(0, 3, 1, 2).cpu()
    assert range_rel_err(got, ref) < 5e-5
    if with_out:
        assert range_rel_err(_join(o_hi, o_lo).permute(0, 3, 1, 2).cpu(), y * s_next[:, :, None, None]) < 5e-5


@pytest.mark.parametrize('N,Cin,Cout,res', [(2, 64, 64, 8), (1, 512, 512, 4), (1, 32, 256, 32), (2, 128, 64, 16), (2, 32, 128, 150)])
def test_upconv_modulated(K, N, Cin, Cout, res):
    """4 transposed-conv parity GEMMs + FIR epilogue == the reference's up=2 modulated conv + bias_act (oracle)."""
    from oracle import ops as oo
    g = _g(17 + res)
    x = torch.randn(N, Cin, res, res, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g)
    s = torch.randn(N, Cin, generator=g)
    b = torch.randn(Cout, generator=g) * 0.1
    nz = torch.randn(2 * res, 2 * res, generator=g) * 0.05
    f = oo.setup_filter()
    ref = oo.bias_act(oo.modulated_conv2d(x, w, s, noise=nz, up=2, padding=1, resample_filter=f, flip_weight=False), b, act='lrelu')
    d = ((w[None] * s[:, None, :, None, None]).square().sum(dim=[2, 3, 4]) + 1e-8).rsqrt()
    a_hi, a_lo = _nhwc_split(K, x * s[:, :, None, None])
    w_hi, w_lo = K.pack_conv_weight(w.to(DEV))
    raw = torch.full((N, 2 * res + 1, 2 * res + 1, Cout), float('nan'), device=DEV)
    for a in (0, 1):                      # the four parity classes as separate launches ...
        for bb in (0, 1):
            K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_transposed(a, bb), N, res + 1 - a, res + 1 - bb, mode=1, out_f32=raw,
                        f32_cstride=Cout, oy_mul=2, oy_off=a, ox_mul=2, ox_off=bb, OH=2 * res + 1, OW=2 * res + 1)
    raw1 = torch.full_like(raw, float('nan'))
    K.conv_transposed_gemm(a_hi, a_lo, w_hi, w_lo, N, res, res, raw1)        # ... and as one multi-class launch
    assert torch.equal(raw, raw1)
    assert not torch.isnan(raw).any()
    out = torch.zeros(N, 2 * res, 2 * res, Cout, device=DEV)
    K.fir_up_epilogue(raw, Cout, d.to(DEV), b.to(DEV), nz.to(DEV), math.sqrt(2), 0.2, -1.0, out_f32=out, f32_cstride=Cout)
    assert range_rel_err(out.permute(0, 3, 1, 2).cpu(), ref) < 3e-5


@pytest.mark.parametrize('per_sample_noise', [False, True], ids=['shared-noise', 'per-sample-noise'])
@pytest.mark.parametrize('N,C,H2', [(3, 128, 256), (3, 256, 128), (5, 512, 64), (5, 64, 256), (1, 128, 512)])
def test_fir_up_streamed_kernel_is_bit_identical(K, N, C, H2, per_sample_noise, monkeypatch):
    """The large layers take the streamed variant (bulk copies of raw rows through a shared-memory ring); it must reproduce the
    register-tiled kernel bit for bit -- fp32 copy, both modulated split-bf16 outputs (one into a concat buffer at a channel offset),
    noise (one map for the batch, or one per image), clamp -- and both must match an fp64 evaluation of upfirdn2d (upfirdn2d.py:120-164,
    pad 1/1, gain 4) + bias_act."""
    g = _g(31 + C + H2)
    raw = torch.randn(N, H2 + 1, H2 + 1, C, generator=g).to(DEV)
    d, b = (torch.rand(N, C, generator=g) + 0.5).to(DEV), torch.randn(C, generator=g).to(DEV)
    nz = (torch.randn(*((N,) if per_sample_noise else ()), H2, H2, generator=g) * 0.1).to(DEV)
    nstride = H2 * H2 if per_sample_noise else 0
    s0, s1 = torch.randn(N, C, generator=g).to(DEV), torch.randn(N, C, generator=g).to(DEV)

    def run(mode):
        monkeypatch.setenv('N3D_FIR_STREAM', mode)
        f32 = torch.zeros(N, H2, H2, C, device=DEV)
        o0 = [torch.zeros(N, H2, H2, C, device=DEV, dtype=torch.bfloat16) for _ in range(2)]
        o1 = [torch.zeros(N, H2, H2, 2 * C, device=DEV, dtype=torch.bfloat16) for _ in range(2)]      # concat buffer, second half
        outs = [K.make_split_out(o0[0], o0[1], s0, C, 0), K.make_split_out(o1[0], o1[1], s1, 2 * C, C)]
        K.fir_up_epilogue(raw, C, d, b, nz, math.sqrt(2), 0.2, 1.5, outs=outs, out_f32=f32, f32_cstride=C, noise_nstride=nstride)
        torch.cuda.synchronize()
        return [f32] + o0 + o1

    a, bb = run('1'), run('0')
    for x, y in zip(a, bb):
        assert torch.equal(x, y)
    f1 = torch.tensor([1., 3., 3., 1.], dtype=torch.float64, device=DEV) / 4
    x = raw.double().permute(0, 3, 1, 2)
    x = F.pad(x, (1, 1, 1, 1))
    y = F.conv2d(x.reshape(N * C, 1, H2 + 3, H2 + 3), torch.outer(f1, f1)[None, None]).reshape(N, C, H2, H2)
    y = y * d.double()[:, :, None, None] + nz.double().reshape(-1, 1, H2, H2) + b.double()[None, :, None, None]
    y = (F.leaky_relu(y, 0.2) * math.sqrt(2)).clamp(-1.5, 1.5)
    assert range_rel_err(a[0].permute(0, 3, 1, 2).cpu(), y.cpu()) < 1e-6
    assert range_rel_err(_join(a[1], a[2]).permute(0, 3, 1, 2).cpu(), (y * s0.double()[:, :, None, None]).cpu()) < 2e-5
    assert range_rel_err(_join(a[3], a[4])[..., C:].permute(0, 3, 1, 2).cpu(), (y * s1.double()[:, :, None, None]).cpu()) < 2e-5
    assert float(a[3][..., :C].abs().max()) == 0.0              # the other half of the concat buffer is untouched


@pytest.mark.parametrize('N,Cin,Cout,res', [(2, 64, 64, 16), (1, 128, 256, 64), (1, 32, 32, 8)])
def test_downconv(K, N, Cin, Cout, res):
    from oracle import ops as oo
    g = _g(19 + res)
    x = torch.randn(N, Cin, res, res, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(Cin * 9)
    b = torch.randn(Cout, generator=g) * 0.1
    ref = oo.bias_act(oo.conv2d_resample(x, w, f=oo.setup_filter(), down=2, padding=1), b, act='lrelu')
    xn = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    SH = (res + 2) // 2
    hi = torch.zeros(4 * N, SH, SH, Cin, device=DEV, dtype=torch.bfloat16)
    lo = torch.zeros_like(hi)
    K.fir_down_split(xn, hi, lo)
    w_hi, w_lo = K.pack_conv_weight(w.to(DEV))
    out = torch.zeros(N, res // 2, res // 2, Cout, device=DEV)
    K.conv_gemm(hi, lo, w_hi, w_lo, K.taps_stride2(), N, res // 2, res // 2, a_img_mul=N, bias=b.to(DEV), gain=math.sqrt(2), slope=0.2,
                out_f32=out, f32_cstride=Cout)
    assert range_rel_err(out.permute(0, 3, 1, 2).cpu(), ref) < 3e-5


@pytest.mark.parametrize('N,C,H', [(3, 128, 256), (4, 256, 128), (8, 512, 64), (8, 64, 128), (2, 128, 250)])
def test_fir_down_streamed_kernel_is_bit_identical(K, N, C, H, monkeypatch):
    """Encoder stride-2 path: the streamed FIR-down kernel (large layers) == the register-tiled one bit for bit (four parity images,
    ragged last row / column tiles, zero padding), and both == an fp64 evaluation of upfirdn2d(pad 2) split by output parity."""
    g = _g(41 + C + H)
    x = torch.randn(N, H, H, C, generator=g).to(DEV)
    SH = (H + 2) // 2

    def run(mode):
        monkeypatch.setenv('N3D_FIR_STREAM', mode)
        hi = torch.full((4 * N, SH, SH, C), 7.0, device=DEV, dtype=torch.bfloat16)
        lo = torch.full_like(hi, 7.0)
        K.fir_down_split(x, hi, lo)
        torch.cuda.synchronize()
        return hi, lo

    (h1, l1), (h0, l0) = run('1'), run('0')
    assert torch.equal(h1, h0) and torch.equal(l1, l0)
    f1 = torch.tensor([1., 3., 3., 1.], dtype=torch.float64, device=DEV) / 8
    xx = F.pad(x.double().permute(0, 3, 1, 2), (2, 2, 2, 2))
    fo = F.conv2d(xx.reshape(N * C, 1, H + 4, H + 4), torch.outer(f1, f1)[None, None]).reshape(N, C, H + 1, H + 1)
    fo = F.pad(fo, (0, 1, 0, 1))                                  # (H+2) x (H+2): the extra row / column is the zero pad
    got = _join(h1, l1).reshape(4, N, SH, SH, C)
    for a in (0, 1):
        for b in (0, 1):
            ref = fo[:, :, a::2, b::2].permute(0, 2, 3, 1)
            assert range_rel_err(got[a * 2 + b].cpu(), ref.cpu()) < 2e-5, (a, b)


# ------------------------------------------------------------------------------------------------ glue kernels
def test_styles_demod(K):
    g = _g(23)
    N, num_ws, cins = 3, 14, [64, 32, 128]
    ws = torch.randn(N, num_ws, 512, generator=g)
    A = torch.randn(sum(cins), 512, generator=g)
    bvec = torch.randn(sum(cins), generator=g)
    widx = torch.cat([torch.full((r,), i + 2, dtype=torch.int32) for i, r in enumerate(cins)])
    scale = torch.cat([torch.full((r,), 1.0 if i != 1 else 0.25) for i, r in enumerate(cins)])
    cin = torch.cat([torch.full((r,), r, dtype=torch.int32) for r in cins])
    base = np.concatenate([[0], np.cumsum(cins)[:-1]])
    ooff = torch.cat([torch.arange(r, dtype=torch.int64) + int(b) * N for r, b in zip(cins, base)])
    ref = torch.stack([(ws[:, widx[r].item()] @ A[r]) / math.sqrt(512) + bvec[r] for r in range(A.shape[0])], 1) * scale[None]
    out = torch.zeros(N * A.shape[0], device=DEV)
    K.styles(ws.to(DEV), A.to(DEV), bvec.to(DEV), widx.to(DEV), scale.to(DEV), ooff.to(DEV), cin.to(DEV), out)
    for r, b in zip(cins, base):
        blk = out[int(b) * N: int(b) * N + N * r].view(N, r).cpu()
        assert range_rel_err(blk, ref[:, int(b): int(b) + r]) < 1e-5
    # demod of a layer with Cin = 64 (first style block) and Cout = 40
    w = torch.randn(40, 64, 3, 3, generator=g)
    wsq = w.square().sum(dim=[2, 3]).reshape(-1)
    dref = ((w[None] * ref[:, None, :64, None, None]).square().sum(dim=[2, 3, 4]) + 1e-8).rsqrt()
    woff = (torch.arange(40, dtype=torch.int64) * 64)
    d = torch.zeros(N * 40, device=DEV)
    K.demod(out, wsq.to(DEV), woff.to(DEV), torch.full((40,), 64, dtype=torch.int32, device=DEV), torch.zeros(40, dtype=torch.int64, device=DEV),
            torch.arange(40, dtype=torch.int64, device=DEV), torch.full((40,), 40, dtype=torch.int32, device=DEV), d, N)
    assert range_rel_err(d.view(N, 40).cpu(), dref) < 1e-5


def test_resample_nhwc(K):
    from oracle import ops as oo
    g = _g(29)
    x = torch.randn(2, 32, 16, 16, generator=g)
    f = oo.setup_filter()
    xn = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    up = torch.zeros(2, 32, 32, 32, device=DEV)
    K.upsample2d_nhwc(xn, up)
    assert range_rel_err(up.permute(0, 3, 1, 2).cpu(), oo.upsample2d(x, f)) < 1e-6
    dn = torch.zeros(2, 8, 8, 32, device=DEV)
    K.downsample2d_nhwc(xn, dn)
    assert range_rel_err(dn.permute(0, 3, 1, 2).cpu(), oo.downsample2d(x, f)) < 1e-6
    s = torch.randn(2, 32, generator=g)
    hi = torch.zeros(2, 16, 16, 32, device=DEV, dtype=torch.bfloat16)
    lo = torch.zeros_like(hi)
    K.modulate_split(xn, s.to(DEV), hi, lo)
    assert range_rel_err(_join(hi, lo).permute(0, 3, 1, 2).cpu(), x * s[:, :, None, None]) < 2e-5


# ------------------------------------------------------------------------------------------------ mesh path
@pytest.fixture(scope='module')
def mesh_case():
    from next3d_b200 import weights
    from oracle import generator as og
    m = weights.load_flame_demo()
    topo = weights.topology_buffers(m)
    v = torch.from_numpy(m['verts'])[None].repeat(2, 1, 1)
    v[1] += torch.randn(v[1].shape, generator=_g(31)) * 2e-4
    lms = torch.from_numpy(m['lms'])[None].repeat(2, 1, 1)
    return dict(mesh=m, topo=topo, v=v, lms=lms, og=og)


def test_transform_and_rasterize_bit_exact(K, mesh_case):
    og, topo, v = mesh_case['og'], mesh_case['topo'], mesh_case['v']
    from oracle import rasterize as orast
    rot = torch.stack([og.angle2matrix(a) for a in og.VIEWS])
    out = torch.zeros(2, 4, 5023, 3, device=DEV)
    K.transform_points(v.to(DEV), rot.to(DEV), 10.0, True, out)
    ref = []
    for view in og.VIEWS:
        tv = og.transform_view(v, view)
        tv[:, :, 2] += 10
        tv[..., :2] = -tv[..., :2]
        ref.append(tv)
    ref = torch.stack(ref, 1)
    assert (out.cpu() - ref).abs().max().item() < 2e-6           # torch.bmm's summation order is not specified: ulp-level
    # bit-exact index buffer on IDENTICAL fp32 vertices (the oracle's)
    faces = topo['faces'][0][:, [0, 2, 1]].to(torch.int32)
    verts = ref.reshape(8, 5023, 3).contiguous()
    p2f_ref, _, bary_ref = orast.rasterize_meshes(verts.numpy(), faces[None].expand(8, -1, -1).numpy(), 256, 256)
    p2f_ref = p2f_ref - (np.arange(8)[:, None, None] * faces.shape[0]) * (p2f_ref >= 0)
    p2f = torch.zeros(8, 256, 256, dtype=torch.int32, device=DEV)
    bary = torch.zeros(8, 256, 256, 3, device=DEV)
    K.rasterize(verts.to(DEV), faces.to(DEV), 256, 256, p2f, bary)
    assert np.array_equal(p2f.cpu().numpy(), p2f_ref.astype(np.int32))
    assert np.array_equal(bary.cpu().numpy(), bary_ref)           # barycentrics bit-identical too
    cov = (p2f[:4] >= 0).float().mean(dim=(1, 2)).cpu()
    assert 0.15 < cov.min().item() and cov.max().item() < 0.4


def test_uv_sample_fill_box(K, mesh_case):
    og, topo, v, lms = mesh_case['og'], mesh_case['topo'], mesh_case['v'], mesh_case['lms']
    g = _g(37)
    N = 2
    tex = torch.randn(N, 32, 256, 256, generator=g)
    mask = torch.ones(1, 1, 256, 256)
    sd = {'faces': topo['faces'], 'face_uvcoords': topo['face_uvcoords']}
    rend, alphas, lm2d, p2fs = og.rasterize(sd, v, lms, tex, mask)
    # device path from the oracle's own transformed vertices (isolates uv_sample / fill_mouth from transform ulps)
    verts = []
    for view in og.VIEWS:
        tv = og.transform_view(v, view)
        tv[:, :, 2] += 10
        tv[..., :2] = -tv[..., :2]
        verts.append(tv)
    verts = torch.stack(verts, 1).reshape(N * 4, 5023, 3).contiguous().to(DEV)
    faces = topo['faces'][0][:, [0, 2, 1]].to(torch.int32).to(DEV)
    face_uv = topo['face_uvcoords'][0][:, [0, 2, 1], :2].contiguous().to(DEV)
    p2f = torch.zeros(N * 4, 256, 256, dtype=torch.int32, device=DEV)
    bary = torch.zeros(N * 4, 256, 256, 3, device=DEV)
    K.rasterize(verts, faces, 256, 256, p2f, bary)
    planes = torch.zeros(3, N, 256, 256, 32, device=DEV)
    alpha = torch.zeros(3, N, 256, 256, device=DEV)
    K.uv_sample(p2f, bary, face_uv, tex.permute(0, 2, 3, 1).contiguous().to(DEV), mask[0, 0].to(DEV), planes, alpha)
    K.fill_mouth(alpha)
    for p in range(3):
        assert range_rel_err(planes[p].permute(0, 3, 1, 2).cpu(), rend[p]) < 1e-5
        assert (alpha[p].cpu() - alphas[p][:, 0]).abs().max().item() < 1e-6
    # mouth box
    lm_t = torch.zeros(N, 4, 68, 3, device=DEV)
    rot = torch.stack([og.angle2matrix(a) for a in og.VIEWS]).to(DEV)
    K.transform_points(lms.to(DEV), rot, 0.0, False, lm_t)
    boxes = torch.zeros(N, 4, dtype=torch.int32, device=DEV)
    K.mouth_box(lm_t[:, 0, :, :2].contiguous(), boxes)
    assert boxes.cpu().tolist() == og.gen_mouth_mask(lm2d[0]).tolist()


def test_fill_mouth_synthetic(K):
    from oracle import generator as og
    a = torch.zeros(3, 1, 64, 64)
    a[:, :, 10:50, 12:52] = 1.0
    a[0, :, 25:30, 20:40] = 0.0
    a[1, :, 20:24, 20:24] = 0.5
    a[1, :, 40:44, 30:34] = 0.0
    a[2, :, :5, :5] = 1.0
    a[2, :, 30:33, 30:36] = 0.0
    # a spiral-ish background channel that needs several sweep iterations
    a[0, :, 55:60, 5:60] = 1.0
    a[0, :, 57, 5:58] = 0.0
    a = (a + F.avg_pool2d(a, 3, 1, 1)) / 2
    ref = og.fill_mouth(a)
    d = a.clone().to(DEV)
    K.fill_mouth(d)
    assert torch.equal(d.cpu(), ref)


@pytest.mark.parametrize('case', ['crop_up', 'paste_down', 'sr_up', 'odd_down'])
def test_resize_aa(K, case):
    g = _g(41)
    if case == 'crop_up':
        src = torch.randn(2, 32, 256, 256, generator=g)
        box = torch.tensor([[82, 122, 108, 148], [80, 133, 100, 153]], dtype=torch.int32)
        ref = torch.cat([F.interpolate(src[i:i + 1, :, b[0]:b[1], b[2]:b[3]], size=(64, 64), mode='bilinear', antialias=True)
                         for i, b in enumerate(box.tolist())])
        dst = torch.zeros(2, 64, 64, 32, device=DEV)
        K.resize_aa(src.permute(0, 2, 3, 1).contiguous().to(DEV), dst, src_box=box.to(DEV))
        assert range_rel_err(dst.permute(0, 3, 1, 2).cpu(), ref) < 1e-5
    elif case == 'paste_down':
        src = torch.randn(2, 32, 256, 256, generator=g)
        base = torch.randn(2, 32, 256, 256, generator=g)
        box = torch.tensor([[82, 122, 108, 148], [60, 113, 90, 143]], dtype=torch.int32)
        ref = base.clone()
        for i, b in enumerate(box.tolist()):
            ref[i:i + 1, :, b[0]:b[1], b[2]:b[3]] = F.interpolate(src[i:i + 1], size=(b[1] - b[0], b[1] - b[0]), mode='bilinear', antialias=True)
        dst = base.permute(0, 2, 3, 1).contiguous().to(DEV)
        K.resize_aa(src.permute(0, 2, 3, 1).contiguous().to(DEV), dst, dst_box=box.to(DEV))
        assert range_rel_err(dst.permute(0, 3, 1, 2).cpu(), ref) < 1e-5
    elif case == 'sr_up':
        src = torch.randn(2, 32, 64, 64, generator=g)
        s = torch.randn(2, 32, generator=g)
        ref = F.interpolate(src, size=(128, 128), mode='bilinear', align_corners=False, antialias=True)
        dst = torch.zeros(2, 128, 128, 32, device=DEV)
        hi = torch.zeros(2, 128, 128, 32, device=DEV, dtype=torch.bfloat16)
        lo = torch.zeros_like(hi)
        K.resize_aa(src.permute(0, 2, 3, 1).contiguous().to(DEV), dst, style=s.to(DEV), hi=hi, lo=lo)
        assert range_rel_err(dst.permute(0, 3, 1, 2).cpu(), ref) < 1e-5
        assert range_rel_err(_join(hi, lo).permute(0, 3, 1, 2).cpu(), ref * s[:, :, None, None]) < 2e-5
    else:
        src = torch.randn(1, 3, 53, 47, generator=g)
        ref = F.interpolate(src, size=(17, 23), mode='bilinear', antialias=True)
        dst = torch.zeros(1, 17, 23, 3, device=DEV)
        K.resize_aa(src.permute(0, 2, 3, 1).contiguous().to(DEV), dst)
        assert range_rel_err(dst.permute(0, 3, 1, 2).cpu(), ref) < 1e-5


def test_blend(K):
    g = _g(43)
    N, H = 2, 32
    front = torch.randn(N, 32, H, H, generator=g)
    tex = torch.randn(N, 3, 32, H, H, generator=g)
    alpha = torch.rand(N, 3, 1, H, H, generator=g)
    stat = torch.randn(N, 96, H, H, generator=g)
    texfull = tex.clone()
    texfull[:, 0] = front
    ref = texfull * alpha + stat.view(N, 3, 32, H, H) * (1 - alpha)
    out = torch.zeros(N, 3, H, H, 32, device=DEV)
    K.blend_planes(front.permute(0, 2, 3, 1).contiguous().to(DEV), tex.permute(1, 0, 3, 4, 2).contiguous().to(DEV),
                   alpha[:, :, 0].permute(1, 0, 2, 3).contiguous().to(DEV), stat.permute(0, 2, 3, 1).contiguous().to(DEV), out)
    assert range_rel_err(out.permute(0, 1, 4, 2, 3).cpu(), ref) < 1e-6


# ------------------------------------------------------------------------------------------------ renderer
@pytest.mark.parametrize('N,res,D,Df,ties', [(2, 32, 48, 48, 0), (1, 16, 96, 96, 0), (1, 24, 36, 36, 0), (1, 20, 48, 0, 0), (1, 16, 40, 24, 0),
                                             (2, 12, 12, 70, 0), (3, 64, 48, 48, 0), (1, 16, 48, 48, 1), (1, 12, 96, 96, 1), (1, 12, 96, 96, 0)])
def test_render_rays(K, N, res, D, Df, ties):
    """Fused renderer vs the oracle with injected sampler noise: both lane layouts (<= 48 / <= 96 samples per pass), ragged tiles,
    image sizes that are not a multiple of the pixel block, coarse-only rendering and unequal coarse / fine resolutions."""
    from next3d_b200 import config, weights
    from oracle import renderer as orr
    cfg = config.tiny_config()
    opts = dict(cfg.rendering_kwargs, depth_resolution=D, depth_resolution_importance=Df)
    g = _g(47 + res)
    planes = torch.randn(N, 3, 32, 64, 64, generator=g)
    sd = {'decoder.net.0.weight': torch.randn(64, 32, generator=g), 'decoder.net.0.bias': torch.randn(64, generator=g) * 0.1,
          'decoder.net.2.weight': torch.randn(33, 64, generator=g), 'decoder.net.2.bias': torch.randn(33, generator=g) * 0.1}
    _, _, c, _ = weights.demo_inputs(cfg, N, seed=5)
    u_c = torch.rand(N, res * res, D, 1, generator=g)
    u_f = torch.rand(N * res * res, max(Df, 1), generator=g)
    if ties:                 # few distinct uniforms: exactly equal fine depths (stable order) and crowded rank buckets (fallback path)
        u_f = torch.floor(u_f * 5) / 5 + 0.01
    cam, intr = c[:, :16].reshape(-1, 4, 4), c[:, 16:25].reshape(-1, 3, 3)
    o, d = orr.ray_sampler(cam, intr, res)
    rgb_ref, depth_ref, w_ref = orr.render(sd, planes, o, d, opts, u_c, u_f)
    dec = ((sd['decoder.net.0.weight'] / math.sqrt(32)).to(DEV).contiguous(), sd['decoder.net.0.bias'].to(DEV),
           (sd['decoder.net.2.weight'] / math.sqrt(64)).to(DEV).contiguous(), sd['decoder.net.2.bias'].to(DEV))
    rgb = torch.zeros(N, res * res, 32, device=DEV)
    depth = torch.zeros(N, res * res, device=DEV)
    wsum = torch.zeros(N, res * res, device=DEV)
    mm = torch.tensor([float('inf'), 0.0], device=DEV)
    K.render_rays(planes.permute(0, 1, 3, 4, 2).contiguous().to(DEV), c[:, :16].contiguous().to(DEV), c[:, 16:25].contiguous().to(DEV), res, opts,
                  dec, rgb, depth, wsum, mm, u_coarse=u_c.to(DEV), u_fine=u_f.to(DEV))
    K.depth_clamp(depth, mm)
    assert range_rel_err(rgb.cpu(), rgb_ref) < 2e-5
    assert range_rel_err(wsum.cpu(), w_ref[..., 0]) < 2e-5
    assert range_rel_err(depth.cpu(), depth_ref[..., 0]) < 2e-5
    # in-kernel RNG: statistically the same image (different noise), finite, inside the valid range
    rgb2 = torch.zeros_like(rgb)
    mm2 = torch.tensor([float('inf'), 0.0], device=DEV)
    K.render_rays(planes.permute(0, 1, 3, 4, 2).contiguous().to(DEV), c[:, :16].contiguous().to(DEV), c[:, 16:25].contiguous().to(DEV), res, opts,
                  dec, rgb2, depth, wsum, mm2, seed=123)
    assert torch.isfinite(rgb2).all() and (rgb2.mean() - rgb.mean()).abs().item() < 0.05


def test_sample_points(K):
    from oracle import renderer as orr
    g = _g(53)
    planes = torch.randn(1, 3, 32, 64, 64, generator=g)
    sd = {'decoder.net.0.weight': torch.randn(64, 32, generator=g), 'decoder.net.0.bias': torch.randn(64, generator=g) * 0.1,
          'decoder.net.2.weight': torch.randn(33, 64, generator=g), 'decoder.net.2.bias': torch.randn(33, generator=g) * 0.1}
    coords = torch.rand(1, 5000, 3, generator=g) * 1.2 - 0.6          # some points fall outside the box (zero padding)
    rgb_ref, sig_ref = orr.run_model(sd, planes, coords, {'box_warp': 1})
    dec = ((sd['decoder.net.0.weight'] / math.sqrt(32)).to(DEV).contiguous(), sd['decoder.net.0.bias'].to(DEV),
           (sd['decoder.net.2.weight'] / math.sqrt(64)).to(DEV).contiguous(), sd['decoder.net.2.bias'].to(DEV))
    sigma = torch.zeros(1, 5000, device=DEV)
    rgb = torch.zeros(1, 5000, 32, device=DEV)
    K.sample_points(planes.permute(0, 1, 3, 4, 2).contiguous().to(DEV), coords.to(DEV), 1.0, dec, sigma, rgb)
    assert range_rel_err(sigma.cpu(), sig_ref[..., 0]) < 3e-5         # decoder on mma.sync, bf16x3 (~2^-16 per product)
    assert range_rel_err(rgb.cpu(), rgb_ref) < 3e-5
