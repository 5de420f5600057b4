"""The fp16 instances of conv_gemm (N3DConvGemm.f16 = 1) and the fp16 single outputs of the epilogue, modulate and resize entry
points, against the contract in include/next3d_b200.h.

The convolution reference is the fp64 product of exactly the fp16 operands the kernel gets (an fp16 x fp16 product is exact in
fp64), so what is left is the fp32 accumulation order and the fp32 epilogue.  Every launch also writes the fp32 output of the same
epilogue values, and an fp16 single output must then equal fp16(fp32 output * style) bit for bit: both are formed from the same fp32
value, one store rounded to fp16.

Every output is a view into a larger allocation filled with a NaN sentinel (tests/helpers.Guarded): the elements a launch owns must
be written, all others must keep the sentinel's bits.

`plan16` mirrors launch_conv's rule for fp16 operands (the bf16 rule with one A and one B tile per stage); the CPU test checks that
the case table reaches every SR launch form, the profiler test that each case ran the conv_gemm_f16_kernel<block_n, block_k> and grid
`plan16` predicts.
"""
import ctypes as C
import re

import pytest
import torch
import torch.nn.functional as F

from tests.helpers import Guarded, launched_kernels, lib, refused

DEV = 'cuda'

# Range-relative bounds, max |got - ref| / max |ref| over the owned elements, with the worst case measured over the table on an
# H100 SXM 80 GB (700 W power limit) beside each.  The fp32 outputs carry only fp32 accumulation and epilogue rounding.
BOUNDS = {'raw': 1e-5,     # worst 1.9e-6 (sr8x_b1conv0_transposed)
          'f32': 3.5e-5,   # worst 6.1e-6 (multi_item_cluster)
          'rgb': 1e-5,     # worst 1.4e-6 (sr8x_b0conv1_rgb256)
          'f16': 6e-4}     # an fp16 output against the fp64 value: half an fp16 ulp (2^-11 = 4.9e-4 of the value) plus the fp32
                           # error; worst 4.34e-4 (sr4x_b0conv1_rgb128)

# ------------------------------------------------------------------------------------------------ the launch rule, mirrored
BLOCK_M, MIN_TILES, MIN_STAGES, MAX_BLOCK_N = 128, 64, 4, 128
EPI_BYTES = max(8 * 128 * 4 + 64 * 36 * 4 + 64 * 4 * 4, 2 * 64 * 32 * 4)
RING_BYTES = 227 * 1024 - 2 * EPI_BYTES - 1024 - 256
BLOCK_NS = (16, 32, 64, 96, 128)


def _pow2_ceil(v):
    p = 1
    while p < v:
        p <<= 1
    return p


def block_k16(Cin, bn):
    """block_k of an fp16 launch: as for bf16, but a stage holds one A and one B tile."""
    return 32 if Cin % 64 == 32 or RING_BYTES // ((BLOCK_M + bn) * 64 * 2) < MIN_STAGES else 64


def plan16(N, Cin, Cout, MH, MW, rgb=False, sms=132, cluster_slots=66):
    """launch_conv's choice for a one-sub-problem fp16 n3d_conv_gemm launch (see tests/test_gpu_conv_conformance.plan)."""
    TW = min(16, _pow2_ceil(MW))
    TH = min(BLOCK_M // TW, _pow2_ceil(MH))
    TN = BLOCK_M // (TW * TH)
    tiles_m = -(-MW // TW) * -(-MH // TH) * -(-N // TN)
    cout16 = -(-Cout // 16) * 16
    bn = next(c for c in (128, 96, 64, 32, 16) if c <= cout16 and (c != 96 or cout16 % 96 == 0))
    while bn > 32 and tiles_m * -(-Cout // bn) < MIN_TILES:
        bn = 32 if bn == 96 else bn // 2
    item_tiles = 1
    if rgb:
        bn = next((w for w in BLOCK_NS if w >= cout16), MAX_BLOCK_N)
        item_tiles = -(-Cout // bn)
    tiles_n = -(-Cout // bn)
    cluster = 2 if bn >= 96 and tiles_m >= 2 else 1
    units = -(-tiles_m // cluster) * tiles_n // item_tiles
    slots = sms if cluster == 1 else cluster_slots
    return dict(block_n=bn, block_k=block_k16(Cin, bn), cluster=cluster, tiles_m=tiles_m, tiles_n=tiles_n, item_tiles=item_tiles,
                grid=cluster * min(units, slots), pad=cluster == 2 and tiles_m % 2 == 1)


# ------------------------------------------------------------------------------------------------ the case table
# The SR launches of the 8XDC head (32 -> 256 -> 128 channels) and the 4X head (32 -> 128 -> 64) at reduced spatial size, plus the
# forms they can take: transposed with the raw TMA store, fused ToRGB over one and two n-tiles, 2-CTA clusters with a pad tile, and
# narrow tiles with an fp16 output into a concat buffer.
def _case(name, N, Cin, Cout, MH, MW, **kw):
    c = dict(name=name, N=N, Cin=Cin, Cout=Cout, MH=MH, MW=MW, transposed=False, rgb=False, outs=None)
    c.update(kw)
    if c['outs'] is None:
        c['outs'] = [] if c['transposed'] else [dict(cstride=Cout, coff=0)]
    return c


CASES = [
    _case('sr8x_b0conv0_transposed', 2, 32, 256, 16, 16, transposed=True),
    _case('sr8x_b0conv1_rgb256', 1, 256, 256, 32, 32, rgb=True),                     # two 128-wide n-tiles per work item
    _case('sr8x_b1conv0_transposed', 1, 256, 128, 16, 16, transposed=True),
    _case('sr8x_b1conv1_rgb128_cluster', 1, 128, 128, 64, 64, rgb=True, outs=[]),    # the last layer: ToRGB only
    _case('sr4x_b0conv0', 2, 32, 128, 32, 32),
    _case('sr4x_b0conv1_rgb128', 1, 128, 128, 32, 32, rgb=True),
    _case('sr4x_b1conv0_transposed', 1, 128, 64, 16, 16, transposed=True),
    _case('sr4x_b1conv1_rgb64', 1, 64, 64, 32, 32, rgb=True),
    _case('pad_tile_cluster', 5, 128, 128, 104, 16, outs=[dict(cstride=128, coff=0), dict(cstride=256, coff=128)]),
    _case('bn16_concat', 2, 64, 16, 16, 16, outs=[dict(cstride=24, coff=8)]),
    _case('bn32_bk32', 1, 96, 40, 8, 16),
    # several work items per CTA (cluster): both consumer warpgroups and the ring's wrap-around, as at the SR's full sizes
    _case('multi_item_cluster', 2, 128, 128, 128, 128),
    _case('multi_item_rgb128', 1, 128, 128, 256, 256, rgb=True, outs=[]),
    _case('multi_item_bn64', 2, 64, 64, 128, 128),
    _case('multi_item_transposed', 2, 256, 128, 64, 64, transposed=True),
]
CASE_IDS = [c['name'] for c in CASES]


def _plan(c):
    if c['transposed']:
        return None                       # nine sub-problems: the instance is checked, not the grid
    return plan16(c['N'], c['Cin'], c['Cout'], c['MH'], c['MW'], rgb=c['rgb'])


def _tiles_m(N, MH, MW):
    TW = min(16, _pow2_ceil(MW))
    TH = min(BLOCK_M // TW, _pow2_ceil(MH))
    return -(-MW // TW) * -(-MH // TH) * -(-N // (BLOCK_M // (TW * TH)))


def _instance(c):
    """(block_n, block_k) of the case's launch.  A transposed launch has nine sub-problems (n3d_conv_transposed_gemm): the four parity
    interiors H x W, two row strips 1 x W, two column strips H x 1 and the corner; block_n follows from their M tiles together."""
    if not c['transposed']:
        p = _plan(c)
        return p['block_n'], p['block_k']
    N, H, W, Cout = c['N'], c['MH'], c['MW'], c['Cout']
    tiles_m = 4 * _tiles_m(N, H, W) + 2 * _tiles_m(N, 1, W) + 2 * _tiles_m(N, H, 1) + _tiles_m(N, 1, 1)
    cout16 = -(-Cout // 16) * 16
    bn = next(x for x in (128, 96, 64, 32, 16) if x <= cout16 and (x != 96 or cout16 % 96 == 0))
    while bn > 32 and tiles_m * -(-Cout // bn) < MIN_TILES:
        bn = 32 if bn == 96 else bn // 2
    return bn, block_k16(c['Cin'], bn)


def test_case_table_covers_every_sr_launch_form():
    """CPU: the table has each form of the SR launches (transposed raw store, fused ToRGB over one and two n-tiles, clusters, a pad
    tile) and both block_k values."""
    plans = {c['name']: _plan(c) for c in CASES if not c['transposed']}
    assert any(c['transposed'] for c in CASES)
    assert any(p['item_tiles'] == 2 for p in plans.values())
    assert any(p['item_tiles'] == 1 and c['rgb'] for c in CASES if not c['transposed'] for p in [plans[c['name']]])
    assert any(p['cluster'] == 2 and c['rgb'] for c in CASES if not c['transposed'] for p in [plans[c['name']]])
    assert any(p['pad'] for p in plans.values())
    assert {p['block_k'] for p in plans.values()} == {32, 64}
    assert {p['block_n'] for p in plans.values()} >= {16, 32, 64, 128}


# ------------------------------------------------------------------------------------------------ one case
def _taps3x3():
    return [(ky - 1, kx - 1, 0, ky * 3 + kx) for ky in range(3) for kx in range(3)]


def _seeded(c):
    g = torch.Generator().manual_seed(sum(map(ord, c['name'])))
    N, Cin, Cout = c['N'], c['Cin'], c['Cout']
    a = (torch.randn(N, c['MH'], c['MW'], Cin, generator=g)).half()
    w = (torch.randn(9, Cout, Cin, generator=g) / (3 * Cin ** 0.5)).half()
    ep = dict(dcoef=torch.rand(N, Cout, generator=g) + 0.5, bias=torch.randn(Cout, generator=g) * 0.1,
              noise=torch.randn(c['MH'], c['MW'], generator=g) * 0.1,
              styles=[torch.rand(N, Cout, generator=g) + 0.5 for _ in c['outs']],
              rgb_w=torch.randn(3, Cout, generator=g), rgb_s=torch.randn(N, Cout, generator=g) / Cout ** 0.5,
              rgb_b=torch.randn(3, generator=g) * 0.1, img=torch.randn(N, 3, c['MH'], c['MW'], generator=g))
    return a, w, ep


def _acc_reference(a, w, transposed):
    """fp64 sum of the exact products of the fp16 operands: a [N,H,W,Cin], w [9,Cout,Cin] -> NHWC."""
    x = a.double().permute(0, 3, 1, 2)
    k = w.double().reshape(3, 3, w.shape[1], w.shape[2])
    if transposed:      # out[2p+a, 2q+b] = sum W[ky,kx] x[p-(ky-a)/2, q-(kx-b)/2] == conv_transpose2d(stride 2), (2H+1) x (2W+1)
        y = F.conv_transpose2d(x, k.permute(3, 2, 0, 1), stride=2)
    else:               # correlation, padding 1, tap (ky, kx) reads x[y + ky - 1, x + kx - 1]
        y = F.conv2d(x, k.permute(2, 3, 0, 1), padding=1)
    return y.permute(0, 2, 3, 1)


def run_case(c):
    """Launch case c -> dict of (Guarded output, reference or None, owned-values check)."""
    from next3d_b200 import kernels as K
    a, w, ep = _seeded(c)
    ad, wd = a.to(DEV), w.to(DEV)
    N, Cout, MH, MW = c['N'], c['Cout'], c['MH'], c['MW']
    acc = _acc_reference(a.to(DEV), w.to(DEV), c['transposed'])
    if c['transposed']:
        raw = Guarded((N, 2 * MH + 1, 2 * MW + 1, Cout))
        K.conv_transposed_gemm(ad, None, wd, None, N, MH, MW, raw.view, nprod=1)
        return dict(raw=(raw, acc, 'raw'))
    d = {k: v.to(DEV) for k, v in ep.items() if k != 'styles'}
    styles = [s.to(DEV).contiguous() for s in ep['styles']]
    v = acc * d['dcoef'].double()[:, None, None, :] + d['noise'].double()[None, :, :, None] + d['bias'].double()
    v = torch.where(v > 0, v, 0.2 * v) * 2 ** 0.5
    v = v.clamp(-1.5, 1.5)
    out = {}
    f32 = Guarded((N, MH, MW, Cout))
    outs, descs = [], []
    for o, s in zip(c['outs'], styles):
        g = Guarded((N, MH, MW, o['cstride']), dtype=torch.float16, own=slice(o['coff'], o['coff'] + Cout))
        outs.append((g, o, s))
        descs.append(K.make_split_out(g.view, None, s, o['cstride'], o['coff'], f16=True))
    rgb = None
    if c['rgb']:
        img = Guarded((N, 3, MH, MW), init=d['img'])
        rgb = dict(out=img.view, weight=d['rgb_w'].contiguous(), style=d['rgb_s'].contiguous(), bias=d['rgb_b'], clamp=2.0, nchw=True,
                   accumulate=True)
        r = torch.einsum('nhwo,co,no->nchw', v, d['rgb_w'].double(), d['rgb_s'].double()) + d['rgb_b'].double()[None, :, None, None]
        out['rgb'] = (img, d['img'].double() + r.clamp(-2.0, 2.0), 'rgb')
    K.conv_gemm(ad, None, wd, None, _taps3x3(), N, MH, MW, nprod=1, dcoef=d['dcoef'], bias=d['bias'], noise=d['noise'], gain=2 ** 0.5,
                slope=0.2, clamp=1.5, outs=descs, out_f32=None if c['rgb'] else f32.view, f32_cstride=Cout, rgb=rgb)
    if not c['rgb']:
        out['f32'] = (f32, v, 'f32')
    for i, (g, o, s) in enumerate(outs):
        out[f'out{i}'] = (g, (f32.view, v, s, o), 'f16')
    return out


def _check(c, out):
    torch.cuda.synchronize()
    errs = {}
    for key, (g, ref, kind) in out.items():
        assert g.untouched_ok(), (c['name'], key, 'wrote outside the elements it owns')
        assert g.written(), (c['name'], key, 'left owned elements unwritten')
        if kind == 'f16':
            f32, v, s, o = ref
            got = g.view[..., o['coff']:o['coff'] + c['Cout']]
            if c['rgb']:            # no fp32 output beside the fused ToRGB: against the fp64 epilogue, within fp16 rounding
                m = v * s.double()[:, None, None, :]
                e = ((got.double() - m).abs().max() / m.abs().max()).item()
                errs[key] = e
                assert e < BOUNDS['f16'], (c['name'], key, e)
            else:
                assert torch.equal(got, (f32 * s[:, None, None, :]).half()), (c['name'], key)
        else:
            e = ((g.view.double() - ref).abs().max() / ref.abs().max()).item()
            errs[key] = e
            assert e < BOUNDS[kind], (c['name'], key, e)
    return errs


@pytest.mark.gpu
@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_conv_gemm_f16_matches_fp64_contract(c):
    errs = _check(c, run_case(c))
    print(c['name'], errs)


@pytest.mark.gpu
def test_launched_f16_instance_matches_plan(tmp_path):
    """Every case under torch.profiler: it launched conv_gemm_f16_kernel<block_n, block_k> as predicted (and, for one-sub-problem
    launches, the predicted grid and cluster)."""
    torch.cuda.synchronize()

    def run():
        for c in CASES:
            run_case(c)
        return CASES

    _, events = launched_kernels(run, r'conv_gemm_f16_kernel', tmp_path)
    props = torch.cuda.get_device_properties(0)
    for c, e in zip(CASES, events):
        m = re.search(r'conv_gemm_f16_kernel<(\d+), (\d+)>', e['name'])
        assert m, e['name']
        inst = _instance(c)
        if inst is not None:
            assert (int(m.group(1)), int(m.group(2))) == inst, (c['name'], e['name'], inst)
        if not c['transposed']:
            p = plan16(c['N'], c['Cin'], c['Cout'], c['MH'], c['MW'], rgb=c['rgb'], sms=props.multi_processor_count,
                       cluster_slots=props.multi_processor_count // 2)
            grid = e.get('args', {}).get('grid')
            if grid is not None:
                assert list(grid) == [p['grid'], 1, 1], (c['name'], grid, p)
            cl = e.get('args', {}).get('cluster')
            if cl is not None:
                assert list(cl)[0] == p['cluster'], (c['name'], cl, p)


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
