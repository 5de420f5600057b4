"""The fused renderer (n3d_render_rays, n3d_render_rays_normals) and the point sampler (n3d_sample_points, n3d_sample_grid) against
the N3DRender contract (include/next3d_b200.h), over a table of small launches that reaches every kernel instance, lane layout and
rendering option the contract offers: white_back, non-square / tiny / production-size planes, box_warp, rays outside the box and
cameras inside it, skewed intrinsics, degenerate densities, the minimum sample counts, uniforms at the ends of [0, 1), ragged pixel
blocks, views and the per-image depth range.  Every case also runs with the in-kernel sampler RNG and must be bit-identical to the
launch fed the host statement's uniforms (tests.helpers.sampler_uniforms), which pins the RNG itself.

Two references, both with the kernel's injected uniforms:
  - oracle.renderer in float32, the pinned statement of the reference's ImportanceRenderer (tests/test_oracle_vs_reference.py,
    test_oracle_long_rays.py, test_oracle_render_contract.py), at the bound of tests/test_gpu_kernels.py::test_render_rays;
  - the same oracle functions evaluated in float64, except in the transparent and opaque cases, where fp32 underflow is the
    contract (softplus(-201) is exactly 0 in fp32, not in fp64).
Every output is a view into a larger allocation filled with a NaN sentinel: every owned element must be written and every guard
element must keep its bits.

`plan` mirrors the work decomposition of make_fused / launch_render (render_fused.cu) in plain Python.  The CPU test checks that the
table covers everything listed in COVERAGE; the profiler test checks on the GPU that each case launched the kernel instance and grid
`plan` predicts.  The alignment tests at the end need no GPU: descriptors over misaligned CPU tensors are refused before any launch.
N3D_RENDER_ERRORS=<file> appends every measured error to <file> as JSON lines, to re-measure the worst cases beside BOUNDS.
"""
import ctypes as C
import math
import re

import pytest
import torch

from tests.helpers import Guarded, launched_kernels, lib, offset_view, range_rel_err, record_errors, refused, sampler_uniforms

DEV = 'cuda'
U_MAX = 1.0 - 2.0 ** -24        # the largest value torch.rand returns

# Range-relative error bounds, max |got - ref| / max |ref| per output.  'oracle': the bound of test_render_rays; 'points': that of
# test_sample_points.  'fp64': kernel against the float64 evaluation, at most 4x the worst case measured over the table on an H100
# 80GB HBM3 (400 W power limit), given beside it.  (reference, case[, output]) keys override them where a case's own rounding
# dominates; the step whose rounding it is stands beside each.
BOUNDS = {
    'oracle': 2e-5,
    'points': 3e-5,
    # opaque: the first interval carries the whole weight, so its colour's unorm16 slot rounding (<= 2^-17, x 2 in the [-1, 1] output)
    # and decoder rounding reach the pixel undiluted instead of averaged over many samples.  Worst 2.6e-5.
    ('oracle', 'opaque', 'rgb'): 6e-5,
    # colour rows of W1 x 100: the sigmoid is 100x steeper, so the bf16x3 decoder's rounding of the colour pre-activation (~1e-6 of
    # |x| <= ~300) moves unsaturated colours by ~1e-5 (the fp32 oracle itself is 3.4e-5 from float64).  Worst 4.2e-5.
    ('oracle', 'saturated_colours', 'rgb'): 1e-4,
    # ray_end - ray_start = 1e-3: every x = sigma * delta is ~1e-4, where the reference's fp32 alpha = 1 - exp(-x) cancels (exp(-x) is
    # within 1e-4 of 1, where its ulp is 6e-8: up to 6e-4 of alpha); the kernel's series for x < 1/16 does not.  The kernel is 2.4e-4
    # from float64 there, the fp32 oracle further.  Worst 6.4e-4 (wsum).
    ('oracle', 'thin_interval', 'wsum'): 2.5e-3,
    'fp64': 3e-5,                                   # worst 8.2e-6 (camera_inside rgb)
    # 256^2 planes: d ix / d x = 256 / box_warp texels per world unit, so the fp32 rounding of a sample position o + t d (~2.4e-7 at
    # the camera's 2.7) moves the bilinear fetch by ~6e-5 texel of unit-variance features; the fp32 oracle itself is 3.6e-5 from
    # float64.  Worst 2.4e-5 (wsum).
    ('fp64', 'planes_256'): 9e-5,
    ('fp64', 'saturated_colours'): 1.5e-4,         # the steep colour sigmoid above; worst 3.8e-5 (rgb)
    # ray_end - ray_start = 1e-3 at t ~ 2.6: fp32 sample depths are quantised to 2.4e-7, 2.6e-3 of the 9.1e-5 coarse spacing, and
    # the float64 evaluation places the samples exactly, so each interval's alpha differs by up to that fraction.  Worst 2.4e-4 (wsum).
    ('fp64', 'thin_interval'): 9.5e-4,
}


def bound(ref, c, out):
    return BOUNDS.get((ref, c['name'], out), BOUNDS.get((ref, c['name']), BOUNDS[ref]))


# ------------------------------------------------------------------------------------------------ the launch rule, mirrored
def lanes(Dc, Df):
    """Lanes per ray (make_fused): 16 up to 48 samples per pass, 32 up to 96, else 64."""
    d = max(Dc, Df)
    return 16 if d <= 48 else 32 if d <= 96 else 64


def plan(N, res, Dc, Df, sms=132):
    """What make_fused / launch_render (render_fused.cu) select for an N-image launch: lanes L, tiles per coarse / fine pass, the
    gw x 2 pixel block of a group of 128 / L rays, groups per image (blocks of 4 x 8 groups, padded), total groups and the grid
    (one persistent CTA per SM, at most one per group)."""
    L = lanes(Dc, Df)
    gw = 64 // L
    tiles_x, tiles_y = -(-res // gw), -(-res // 2)
    blocks_x = -(-tiles_x // 4)
    gpi = blocks_x * -(-tiles_y // 8) * 32
    total = N * gpi
    return dict(L=L, Tc=-(-Dc // L), Tf=-(-Df // L), gw=gw, gpi=gpi, total_groups=total, grid=min(total, sms),
                ragged=res % gw != 0 or res % 2 != 0)


def normals_grid(N, res, sms=132):
    """launch_normals: one warp per ray, 8 warps per CTA, at most two CTAs per SM."""
    return min(-(-(N * res * res) // 8), 2 * sms)


def points_grid(N, Pn, sms=132):
    """launch_points: 128-point tiles, at most one CTA per SM."""
    return min(-(-(N * Pn) // 128), sms)


# ------------------------------------------------------------------------------------------------ the case table
def _case(name, axis, **kw):
    c = dict(name=name, axis=axis, N=1, res=12, Dc=12, Df=12, PH=64, PW=64, box_warp=1.0, ray_start=2.25, ray_end=3.3,
             white_back=False, camera='demo', density='mid', uniforms='random', views=1, per_image=0, normals=False, seed_ptr=False)
    c.update(kw)
    return c


CASES = [
    # lane layouts, fine and coarse-only; res not a multiple of the pixel block (4 x 2, 2 x 2, 1 x 2) leaves ragged groups
    _case('l16_fine', 'lanes', res=13, Dc=40, Df=24, normals=True),
    _case('l16_coarse_only', 'lanes', res=13, Dc=48, Df=0),
    _case('l32_fine', 'lanes', res=11, Dc=64, Df=80, normals=True, seed_ptr=True),
    _case('l32_coarse_only', 'lanes', res=9, Dc=96, Df=0),
    _case('l64_fine', 'lanes', res=7, Dc=100, Df=150, normals=True),
    _case('l64_coarse_only', 'lanes', res=6, Dc=192, Df=0),
    # white_back in every layout, with and without fine samples (with views and the per-image depth range on some)
    _case('white_l16_fine', 'white_back', res=10, Dc=24, Df=48, white_back=True),
    _case('white_l16_coarse_only', 'white_back', res=10, Dc=48, Df=0, white_back=True, N=2, per_image=1),
    _case('white_l32_fine', 'white_back', res=8, Dc=96, Df=49, white_back=True, N=4, views=2, per_image=1, seed_ptr=True),
    _case('white_l32_coarse_only', 'white_back', res=8, Dc=49, Df=0, white_back=True),
    _case('white_l64_fine', 'white_back', res=5, Dc=97, Df=120, white_back=True, N=2, views=2),
    _case('white_l64_coarse_only', 'white_back', res=5, Dc=150, Df=0, white_back=True),
    # planes: PH != PW both ways, 5 x 3 (most taps on the border), production 256^2, several plane sets
    _case('planes_48x80', 'planes', PH=48, PW=80, normals=True),
    _case('planes_80x48', 'planes', PH=80, PW=48, normals=True, N=3, views=3),
    _case('planes_5x3', 'planes', PH=5, PW=3, normals=True),
    _case('planes_256', 'planes', PH=256, PW=256, res=16),
    _case('planes_n3_per_image', 'planes', N=3, PH=24, PW=40, per_image=1),
    # box
    _case('box_warp_0.5', 'box', box_warp=0.5, normals=True),
    _case('box_warp_3', 'box', box_warp=3.0),
    # ray interval: every sample outside the box (all taps zero-padded), camera inside the box, a 1e-3 interval
    _case('beyond_box', 'ray interval', ray_start=4.0, ray_end=5.0),
    _case('camera_inside', 'ray interval', camera='inside', ray_start=0.01, ray_end=1.2, normals=True),
    _case('thin_interval', 'ray interval', ray_start=2.6, ray_end=2.601),
    # cameras
    _case('skewed_intrinsics', 'cameras', camera='skewed', normals=True),
    _case('cam2world_bottom_row', 'cameras', camera='bottom_row'),
    # densities
    _case('transparent', 'densities', density='transparent', N=2),
    _case('transparent_white_back', 'densities', density='transparent', white_back=True, Df=0, N=2, per_image=1),
    _case('opaque', 'densities', density='opaque'),
    _case('saturated_colours', 'densities', density='saturated'),
    # the minimum sample counts check_render accepts, one fine sample at 192 coarse
    _case('dc4_df0', 'sample counts', Dc=4, Df=0),
    _case('dc4_df1', 'sample counts', Dc=4, Df=1, uniforms='edges'),
    _case('dc5_df2', 'sample counts', Dc=5, Df=2),
    _case('dc192_df1', 'sample counts', res=6, Dc=192, Df=1),
    # uniforms exactly 0 and 1 - 2^-24 mixed with random ones
    _case('uniform_edges_l16', 'uniforms', Dc=24, Df=24, uniforms='edges'),
    _case('uniform_edges_l64', 'uniforms', res=6, Dc=150, Df=150, uniforms='edges'),
    # schedule: one ray per image, several times more groups than SMs
    _case('res1_n3', 'schedule', res=1, N=3),
    _case('many_groups', 'schedule', res=64, N=2, Dc=12, Df=12),
]
CASE_IDS = [c['name'] for c in CASES]
NORMAL_CASES = [c for c in CASES if c['normals']]


def _plan(c, sms=132):
    return plan(c['N'], c['res'], c['Dc'], c['Df'], sms)


COVERAGE = {
    'every lane layout with fine samples and coarse-only':
        lambda cs: {(p['L'], c['Df'] > 0) for c, p in cs} >= {(L, f) for L in (16, 32, 64) for f in (False, True)},
    'white_back in every lane layout with fine samples and coarse-only':
        lambda cs: {(p['L'], c['Df'] > 0) for c, p in cs if c['white_back']} >= {(L, f) for L in (16, 32, 64) for f in (False, True)},
    'ragged pixel blocks in every lane layout': lambda cs: {p['L'] for c, p in cs if p['ragged']} == {16, 32, 64},
    'PH != PW both ways': lambda cs: {(48, 80), (80, 48)} <= {(c['PH'], c['PW']) for c, p in cs},
    'tiny odd planes': lambda cs: any(c['PH'] * c['PW'] <= 16 and c['PH'] % 2 and c['PW'] % 2 for c, p in cs),
    'production 256^2 planes': lambda cs: any(c['PH'] == c['PW'] == 256 for c, p in cs),
    'several plane sets': lambda cs: any(c['N'] // c['views'] >= 2 for c, p in cs),
    'box_warp 0.5 and 3': lambda cs: {0.5, 3.0} <= {c['box_warp'] for c, p in cs},
    'ray interval beyond the box': lambda cs: any(c['ray_start'] - 2.7 > math.sqrt(3) * c['box_warp'] / 2 for c, p in cs),
    'camera inside the box': lambda cs: any(c['camera'] == 'inside' and c['ray_start'] <= 0.01 for c, p in cs),
    'ray interval of 1e-3': lambda cs: any(abs(c['ray_end'] - c['ray_start'] - 1e-3) < 1e-6 for c, p in cs),
    'skewed off-centre intrinsics': lambda cs: any(c['camera'] == 'skewed' for c, p in cs),
    'non-zero bottom row in cam2world': lambda cs: any(c['camera'] == 'bottom_row' for c, p in cs),
    'transparent, with and without white_back': lambda cs: {False, True} <= {c['white_back'] for c, p in cs if c['density'] == 'transparent'},
    'opaque and saturated colours': lambda cs: {'opaque', 'saturated'} <= {c['density'] for c, p in cs},
    'sample counts (4, 0), (4, 1), (5, 2), (192, 1)': lambda cs: {(4, 0), (4, 1), (5, 2), (192, 1)} <= {(c['Dc'], c['Df']) for c, p in cs},
    'uniforms at the ends of [0, 1) in two lane layouts': lambda cs: len({p['L'] for c, p in cs if c['uniforms'] == 'edges'}) >= 2,
    'res 1 with N 3': lambda cs: any(c['res'] == 1 and c['N'] == 3 for c, p in cs),
    'several times more groups than SMs': lambda cs: any(p['total_groups'] >= 4 * 132 for c, p in cs),
    'one CTA per group (fewer groups than SMs)': lambda cs: any(p['total_groups'] < 132 for c, p in cs),
    'depth range: per image and global, views 1 and >= 2':
        lambda cs: {(c['per_image'], c['views'] >= 2) for c, p in cs} >= {(a, b) for a in (0, 1) for b in (False, True)},
    'normals in every lane layout': lambda cs: {p['L'] for c, p in cs if c['normals']} == {16, 32, 64},
    'normals on non-square, 5 x 3, box_warp 0.5, skewed and inside-the-box geometry':
        lambda cs: {'planes_48x80', 'planes_80x48', 'planes_5x3', 'box_warp_0.5', 'skewed_intrinsics', 'camera_inside'}
        <= {c['name'] for c, p in cs if c['normals']},
    'the in-kernel RNG through seed_ptr, with normals and with views and the per-image depth range':
        lambda cs: any(c['seed_ptr'] and c['normals'] for c, p in cs) and any(c['seed_ptr'] and c['views'] >= 2 and c['per_image'] for c, p in cs),
}


def test_case_table_covers_every_configuration():
    """CPU: the table reaches everything listed in COVERAGE, according to the mirrored launch rule; every case names its axis."""
    planned = [(c, _plan(c)) for c in CASES]
    missing = [k for k, ok in COVERAGE.items() if not ok(planned)]
    assert not missing, missing
    assert len(set(CASE_IDS)) == len(CASE_IDS)
    assert all(c['axis'] for c in CASES)
    assert all(c['N'] % c['views'] == 0 for c in CASES)


# ------------------------------------------------------------------------------------------------ inputs and references
def _decoder(density, g):
    sd = {'decoder.net.0.weight': torch.randn(64, 32, generator=g), 'decoder.net.0.bias': torch.randn(64, generator=g) * 0.1,
          'decoder.net.2.weight': torch.randn(33, 64, generator=g), 'decoder.net.2.bias': torch.randn(33, generator=g) * 0.1}
    if density == 'transparent':                # sigma = -200 exactly: softplus(-201) underflows to 0, every weight is 0
        sd['decoder.net.2.weight'][0] = 0
        sd['decoder.net.2.bias'][0] = -200.0
    elif density == 'opaque':                   # alpha = 1 on the first interval
        sd['decoder.net.2.bias'][0] = 1e4
    elif density == 'saturated':                # sigmoid colours at 0 and 1: the unorm16 colour slots hit 0 and 65535
        sd['decoder.net.2.weight'][1:] *= 100
    return sd


def _dec(sd):
    return ((sd['decoder.net.0.weight'] / math.sqrt(32)).to(DEV).contiguous(), sd['decoder.net.0.bias'].to(DEV),
            (sd['decoder.net.2.weight'] / math.sqrt(64)).to(DEV).contiguous(), sd['decoder.net.2.bias'].to(DEV))


def _cameras(c, g):
    """cam2world [N, 4, 4], intrinsics [N, 3, 3] of a case."""
    from next3d_b200 import config, weights
    _, _, cams, _ = weights.demo_inputs(config.tiny_config(), c['N'], seed=5)
    cam2world, intr = cams[:, :16].reshape(-1, 4, 4).clone(), cams[:, 16:25].reshape(-1, 3, 3).clone()
    if c['camera'] == 'skewed':                 # skew, fx != fy, cx != cy != 0.5
        intr[:, 0, 0], intr[:, 0, 1], intr[:, 0, 2], intr[:, 1, 1], intr[:, 1, 2] = 4.0, 0.35, 0.46, 4.5, 0.57
    elif c['camera'] == 'bottom_row':           # the contract reads the top three rows only
        cam2world[:, 3] = torch.tensor([0.25, -0.5, 0.75, 2.0])
    elif c['camera'] == 'inside':               # the demo orientations, placed inside the [-0.5, 0.5]^3 box
        cam2world[:, :3, 3] = torch.tensor([0.1, -0.05, 0.15]) + 0.02 * torch.randn(c['N'], 3, generator=g)
    return cam2world, intr


def _edges(u, g):
    """A quarter of the uniforms set to exactly 0, a quarter to 1 - 2^-24."""
    r = torch.rand(u.shape, generator=g)
    u[r < 0.25] = 0.0
    u[r > 0.75] = U_MAX
    return u


def setup_case(c):
    """Inputs of a case (CPU; the oracle's layouts): opts, planes [B, 3, 32, PH, PW], sd, cam2world, intrinsics, u_coarse, u_fine."""
    from next3d_b200 import config
    g = torch.Generator().manual_seed(3000 + CASE_IDS.index(c['name']))
    N, res, Dc, Df = c['N'], c['res'], c['Dc'], c['Df']
    opts = dict(config.tiny_config().rendering_kwargs, depth_resolution=Dc, depth_resolution_importance=Df, box_warp=c['box_warp'],
                ray_start=c['ray_start'], ray_end=c['ray_end'], white_back=c['white_back'])
    planes = torch.randn(N // c['views'], 3, 32, c['PH'], c['PW'], generator=g)
    sd = _decoder(c['density'], g)
    cam2world, intr = _cameras(c, g)
    u_c = torch.rand(N, res * res, Dc, 1, generator=g)
    u_f = torch.rand(N * res * res, max(Df, 1), generator=g)
    if c['uniforms'] == 'edges':
        _edges(u_c, g)
        _edges(u_f, g)
    return dict(c=c, opts=opts, planes=planes, sd=sd, cam2world=cam2world, intr=intr, u_c=u_c, u_f=u_f)


def oracle(s, dtype=torch.float32):
    """oracle.renderer on the case in `dtype` -> rgb [N, M, 32], depth [N, M] (clamped), wsum [N, M], depth_minmax ([2] or [N, 2]).
    Per-image depth range: every image rendered on its own, as the contract describes it."""
    from oracle import renderer as orr
    c = s['c']
    N, M = c['N'], c['res'] ** 2
    planes = s['planes'].repeat_interleave(c['views'], 0).to(dtype)
    sd = {k: v.to(dtype) for k, v in s['sd'].items()}
    o, d = orr.ray_sampler(s['cam2world'].to(dtype), s['intr'].to(dtype), c['res'])
    u_c, u_f = s['u_c'].to(dtype), s['u_f'].to(dtype)
    parts = [range(N)] if not c['per_image'] else [range(n, n + 1) for n in range(N)]
    out = []
    for r in parts:
        a, b = r.start, r.stop
        rgb, depth, wsum, t = orr.render(sd, planes[a:b], o[a:b], d[a:b], s['opts'], u_c[a:b], u_f[a * M:b * M], return_depths=True)
        out.append((rgb, depth[..., 0], wsum[..., 0], torch.stack([t.min(), t.max()])))
    rgb, depth, wsum = (torch.cat([x[i] for x in out]) for i in range(3))
    mm = torch.stack([x[3] for x in out]) if c['per_image'] else out[0][3]
    return rgb, depth, wsum, mm


def _outputs(c):
    N, M = c['N'], c['res'] ** 2
    init = torch.tensor([float('inf'), float('-inf')], device=DEV)
    mm = Guarded((N, 2), init=init.expand(N, 2)) if c['per_image'] else Guarded((2,), init=init)
    return dict(rgb=Guarded((N, M, 32)), depth=Guarded((N, M)), wsum=Guarded((N, M)), mm=mm)


def _device_inputs(s, planes=None):
    c = s['c']
    pl = (s['planes'] if planes is None else planes).permute(0, 1, 3, 4, 2).contiguous().to(DEV)
    return dict(planes=pl, cam=s['cam2world'].reshape(c['N'], 16).to(DEV), intr=s['intr'].reshape(c['N'], 9).to(DEV),
                dec=_dec(s['sd']), u_c=s['u_c'].to(DEV), u_f=s['u_f'].to(DEV))


def launch_case(s, out, dv=None, views=None, normal=None, work=None, seed=0, seed_ptr=None):
    """n3d_render_rays (or n3d_render_rays_normals with normal / work) with injected uniforms (the in-kernel RNG with `seed` and
    `seed_ptr` where dv's are None), then the depth clamp."""
    from next3d_b200 import kernels as K
    c = s['c']
    dv = dv or _device_inputs(s)
    args = (dv['planes'], dv['cam'], dv['intr'], c['res'], s['opts'], dv['dec'], out['rgb'].view, out['depth'].view, out['wsum'].view,
            out['mm'].view)
    kw = dict(u_coarse=dv['u_c'], u_fine=dv['u_f'], views=c['views'] if views is None else views, depth_range_per_image=c['per_image'],
              seed=seed, seed_ptr=seed_ptr)
    if normal is None:
        K.render_rays(*args, **kw)
    else:
        K.render_rays_normals(*args, normal, work, **kw)
    if c['per_image']:
        K.depth_clamp_images(out['depth'].view, out['mm'].view)
    else:
        K.depth_clamp(out['depth'].view, out['mm'].view)


# ------------------------------------------------------------------------------------------------ n3d_render_rays
@pytest.mark.gpu
@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_render_rays_matches_contract(c):
    s = setup_case(c)
    out = _outputs(c)
    dv = _device_inputs(s)
    launch_case(s, out, dv)
    torch.cuda.synchronize()
    for k, g in out.items():
        assert g.untouched_ok(), f'{k}: an element outside the output was written'
        assert g.written(), f'{k}: an owned element was not written'
    rgb, depth, wsum, mm = (out[k].view.cpu() for k in ('rgb', 'depth', 'wsum', 'mm'))
    assert torch.isfinite(rgb).all() and torch.isfinite(depth).all() and torch.isfinite(wsum).all() and torch.isfinite(mm).all()

    ref = oracle(s)
    errs = {k: range_rel_err(x, r) for k, x, r in zip(('rgb', 'depth', 'wsum', 'depth_minmax'), (rgb, depth, wsum, mm), ref)}
    if c['density'] == 'transparent':           # every weight is 0: wsum 0, background colour, depth clamped to the launch's far end
        assert not wsum.any() and not ref[2].any()
        assert (rgb == (1.0 if c['white_back'] else -1.0)).all()
        far = mm[:, 1:] if c['per_image'] else mm[1]
        assert torch.equal(depth, far.expand_as(depth))
    record_errors('N3D_RENDER_ERRORS', [{'kind': 'oracle', 'case': c['name'], **errs}])
    bad = {k: e for k, e in errs.items() if not e < bound('oracle', c, k)}
    if c['density'] not in ('transparent', 'opaque'):
        ref64 = oracle(s, torch.float64)
        errs64 = {k: range_rel_err(x, r) for k, x, r in zip(('rgb', 'depth', 'wsum'), (rgb, depth, wsum), ref64)}
        record_errors('N3D_RENDER_ERRORS', [{'kind': 'fp64', 'case': c['name'], **errs64}])
        bad.update({f'fp64 {k}': e for k, e in errs64.items() if not e < bound('fp64', c, k)})
    assert not bad, bad

    if c['views'] >= 2:                         # bit for bit the launch on the plane sets repeated `views` times
        rep = _outputs(c)
        launch_case(s, rep, _device_inputs(s, s['planes'].repeat_interleave(c['views'], 0)), views=1)
        for k in out:
            assert torch.equal(out[k].view, rep[k].view), k


# ------------------------------------------------------------------------------------------------ the in-kernel sampler RNG
def rng_seeds(c):
    """(descriptor seed, *seed_ptr or None) of a case's in-kernel RNG launch: seeds with high bits set, split between the two fields
    (which the kernel adds modulo 2^64) in the seed_ptr cases."""
    seed = 0xC3A5C85C97CB3127 + CASE_IDS.index(c['name'])
    return (0x9AE16A3B2F90404F, (seed - 0x9AE16A3B2F90404F) % 2 ** 64) if c['seed_ptr'] else (seed, None)


@pytest.mark.gpu
@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_in_kernel_rng_matches_host_statement(c):
    """u_coarse = u_fine = None with a seed == the same launch fed tests.helpers.sampler_uniforms of that seed, bit for bit, in every
    output (n3d_render_rays_normals in the normal cases, its normals and exported samples included).  seed_ptr cases: the kernel's
    seed is the descriptor's plus *seed_ptr, read as uint64."""
    from next3d_b200 import kernels as K
    s = setup_case(c)
    N, M = c['N'], c['res'] ** 2
    seed, extra = rng_seeds(c)
    u_c, u_f = sampler_uniforms(seed + (extra or 0), N, M, c['Dc'], c['Df'])         # the statement takes the sum modulo 2^64
    dv = _device_inputs(s)
    runs = []
    for inject in (True, False):
        out = _outputs(c)
        kw = {}
        if c['normals']:
            out['normal'] = Guarded((N, M, 3))
            out['work'] = Guarded((K.normals_workspace_floats(N, c['res'], s['opts']),))
            kw = dict(normal=out['normal'].view, work=out['work'].view)
        if inject:
            launch_case(s, out, dict(dv, u_c=u_c.to(DEV), u_f=u_f.to(DEV)), **kw)
        else:
            ptr = None if extra is None else torch.tensor([extra - 2 ** 64 if extra >> 63 else extra], dtype=torch.int64, device=DEV)
            launch_case(s, out, dict(dv, u_c=None, u_f=None), seed=seed, seed_ptr=ptr, **kw)
        runs.append(out)
    torch.cuda.synchronize()
    for k in runs[0]:
        assert runs[1][k].untouched_ok() and runs[1][k].written(), k
        assert torch.equal(runs[0][k].snapshot(), runs[1][k].snapshot()), k


# ------------------------------------------------------------------------------------------------ n3d_render_rays_normals
@pytest.mark.gpu
@pytest.mark.parametrize('c', NORMAL_CASES, ids=[c['name'] for c in NORMAL_CASES])
def test_render_rays_normals_matches_contract(c):
    """rgb / depth / wsum / depth range bit-identical to n3d_render_rays; the exported samples and the normals against the oracle with
    the criteria of tests/test_gpu_normals.py."""
    from next3d_b200 import kernels as K
    from oracle import normals as onr, renderer as orr
    from tests.test_gpu_normals import _check_against_oracle
    s = setup_case(c)
    N, M = c['N'], c['res'] ** 2
    dv = _device_inputs(s)
    a, b = _outputs(c), _outputs(c)
    launch_case(s, a, dv)
    normal = Guarded((N, M, 3))
    work = Guarded((K.normals_workspace_floats(N, c['res'], s['opts']),))
    launch_case(s, b, dv, normal=normal.view, work=work.view)
    torch.cuda.synchronize()
    for k in a:
        assert torch.equal(a[k].view, b[k].view), k
    assert normal.untouched_ok() and normal.written() and work.untouched_ok() and work.written()
    planes = s['planes'].repeat_interleave(c['views'], 0)
    o, d = orr.ray_sampler(s['cam2world'], s['intr'], c['res'])
    ref = onr.render_normals(s['sd'], planes, o, d, s['opts'], s['u_c'], s['u_f'], return_samples=True)
    _check_against_oracle(s['sd'], planes, o, d, s['opts'], work.view.view(N, M, -1), normal.view, ref)


@pytest.mark.gpu
def test_coarse_depths_follow_the_double_spacing():
    """Coarse-only rendering exports the jittered coarse depths themselves: linspace(ray_start, ray_end) + u * spacing, with the
    spacing (ray_end - ray_start) / (Dc - 1) formed from the caller's double endpoints as the reference does.  On a 1e-3 interval at
    t = 2.6, a spacing formed from the descriptor's float endpoints is 1.7e-4 off, which moves about one coarse depth in 30 by an
    ulp.  What may remain is the kernel's fused multiply-add against the reference's rounded product, which moves a depth only when
    u * spacing sits within its own ulp of a rounding boundary (about 2e-4 of them here)."""
    from next3d_b200 import config, kernels as K
    from oracle import renderer as orr
    ray_start, ray_end, Dc = 2.6, 2.601, 12
    N, res = 2, 16
    M = res * res
    opts = dict(config.tiny_config().rendering_kwargs, depth_resolution=Dc, depth_resolution_importance=0, ray_start=ray_start,
                ray_end=ray_end)
    g = torch.Generator().manual_seed(4200 + Dc)
    s = dict(c=dict(N=N, res=res, views=1, per_image=0), opts=opts, planes=torch.randn(N, 3, 32, 16, 16, generator=g),
             sd=_decoder('mid', g), u_c=torch.rand(N, M, Dc, 1, generator=g), u_f=torch.rand(N * M, 1, generator=g))
    s['cam2world'], s['intr'] = _cameras(dict(N=N, camera='demo'), g)
    out = _outputs(s['c'])
    work = torch.full((K.normals_workspace_floats(N, res, opts),), float('nan'), device=DEV)
    launch_case(s, out, normal=torch.empty(N, M, 3, device=DEV), work=work)
    o, d = orr.ray_sampler(s['cam2world'], s['intr'], res)
    t_ref = orr.render(s['sd'], s['planes'], o, d, opts, s['u_c'], s['u_f'], return_depths=True)[3]
    t = work.view(N, M, 2 * Dc - 1)[..., :Dc].cpu()
    moved = (t != t_ref).double().mean().item()
    assert (t - t_ref).abs().max().item() <= 2.5e-7 and moved <= 2e-3, moved


# ------------------------------------------------------------------------------------------------ n3d_sample_points / n3d_sample_grid
POINT_CASES = [
    dict(name='n3_pn1000_tiles_straddle_sets', N=3, Pn=1000, PH=64, PW=64, box_warp=1.0, rgb=True, special=False),
    dict(name='rgb_null', N=2, Pn=1000, PH=64, PW=64, box_warp=1.0, rgb=False, special=False),
    dict(name='planes_48x80_box_0.5_edges', N=2, Pn=0, PH=48, PW=80, box_warp=0.5, rgb=True, special=True),
]


def _special_coords(PH, PW, box_warp, g):
    """Points exactly at +-box_warp / 2, on texel centres and on bilinear cell edges of every plane (ix = ((x + 1) * W - 1) / 2 is an
    integer on a centre, an integer + 1/2 on an edge), with the third coordinate random inside and just outside the box."""
    h = box_warp / 2
    vals = []
    for size in (PW, PH):
        i = torch.arange(-1, size + 1, dtype=torch.float64)
        vals += [((2 * i + 1) / size - 1) * h, ((2 * i + 2) / size - 1) * h]       # centres, edges (incl. one beyond each border)
    vals = torch.cat(vals + [torch.tensor([-h, h, 0.0], dtype=torch.float64)]).float()
    n = vals.numel()
    pts = []
    for axis in range(3):                        # the special value on each axis in turn
        p = (torch.rand(n, 3, generator=g) * 2 - 1) * h * 1.1
        p[:, axis] = vals
        pts.append(p)
    corners = torch.tensor([[sx * h, sy * h, sz * h] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)])
    return torch.cat(pts + [corners])


def _points_setup(pc):
    g = torch.Generator().manual_seed(4000 + [p['name'] for p in POINT_CASES].index(pc['name']))
    planes = torch.randn(pc['N'], 3, 32, pc['PH'], pc['PW'], generator=g)
    sd = _decoder('mid', g)
    if pc['special']:
        coords = torch.stack([_special_coords(pc['PH'], pc['PW'], pc['box_warp'], g) for _ in range(pc['N'])])
    else:
        coords = (torch.rand(pc['N'], pc['Pn'], 3, generator=g) * 2 - 1) * pc['box_warp'] * 0.6
    return planes, sd, coords


def launch_points(pc, planes, sd, coords):
    from next3d_b200 import kernels as K
    N, Pn = coords.shape[:2]
    sigma = Guarded((N, Pn))
    rgb = Guarded((N, Pn, 32)) if pc['rgb'] else None
    K.sample_points(planes.permute(0, 1, 3, 4, 2).contiguous().to(DEV), coords.to(DEV), pc['box_warp'], _dec(sd), sigma.view,
                    rgb.view if rgb else None)
    return sigma, rgb


@pytest.mark.gpu
@pytest.mark.parametrize('pc', POINT_CASES, ids=[p['name'] for p in POINT_CASES])
def test_sample_points_matches_oracle(pc):
    from oracle import renderer as orr
    planes, sd, coords = _points_setup(pc)
    sigma, rgb = launch_points(pc, planes, sd, coords)
    torch.cuda.synchronize()
    rgb_ref, sig_ref = orr.run_model(sd, planes, coords, {'box_warp': pc['box_warp']})
    errs = {}
    for name, g, ref in (('sigma', sigma, sig_ref[..., 0]), ('rgb', rgb, rgb_ref)):
        if g is None:
            continue
        assert g.untouched_ok() and g.written(), name
        errs[name] = range_rel_err(g.view.cpu(), ref)
    record_errors('N3D_RENDER_ERRORS', [{'kind': 'points', 'case': pc['name'], **errs}])
    assert all(e < BOUNDS['points'] for e in errs.values()), errs


@pytest.mark.gpu
def test_sample_grid_non_square_planes_box_0_5():
    """n3d_sample_grid on 48 x 80 planes with box_warp 0.5 (most voxels of the unit cube outside the box) == oracle run_model on the
    create_samples coordinates, then the script's flip + trim (as tests/test_gpu_drivers.py does for square planes)."""
    from next3d_b200 import drivers, kernels as K
    from oracle import renderer as orr
    R = 40
    g = torch.Generator().manual_seed(4100)
    planes = torch.randn(1, 3, 32, 48, 80, generator=g)
    sd = _decoder('mid', g)
    pad = int(30 * R / 256)
    _, sig_ref = orr.run_model(sd, planes, drivers.create_samples(R, 1.0), {'box_warp': 0.5})
    ref = drivers.trim_sigma_grid(sig_ref.reshape(R, R, R).clone(), R)
    out = Guarded((R, R, R))
    K.sample_grid(planes.permute(0, 1, 3, 4, 2).contiguous().to(DEV)[0], R, 1.0, 0.5, _dec(sd), out.view, pad=pad)
    torch.cuda.synchronize()
    assert out.untouched_ok() and out.written()
    got = out.view.cpu()
    border = ref == -1000.0
    assert border.any() and torch.equal(got[border], ref[border])
    err = range_rel_err(got[~border], ref[~border])
    record_errors('N3D_RENDER_ERRORS', [{'kind': 'grid', 'case': 'planes_48x80_box_0.5', 'sigma': err}])
    assert err < BOUNDS['points'], err


# ------------------------------------------------------------------------------------------------ 32-bit texel offsets
@pytest.mark.gpu
def test_plane_sets_at_the_end_of_32_bit_texel_offsets():
    """170 plane sets at 256^2 (4.28 GB, just under the 2^32-byte limit of the uint32 texel offsets of all three kernels), every set
    different: n3d_render_rays at N = 170 and at views = 2 (N = 340), n3d_render_rays_normals and n3d_sample_points, sets 0, 84 and
    169 against the oracle."""
    from next3d_b200 import config, kernels as K, weights
    from oracle import normals as onr, renderer as orr
    from tests.test_gpu_normals import _check_against_oracle
    B, P, res = 170, 256, 2
    assert B * 3 * P * P * 128 < 2 ** 32 < (B + 1) * 3 * P * P * 128
    planes = torch.empty(B, 3, P, P, 32, device=DEV)            # channels-last, as the kernels read it
    for i in range(B):
        planes[i].normal_(generator=torch.Generator(device=DEV).manual_seed(5000 + i))
    check = [0, 84, 169]
    host = planes[check].permute(0, 1, 4, 2, 3).cpu()               # [3, 3, 32, P, P] in the oracle's layout
    g = torch.Generator().manual_seed(5200)
    sd = _decoder('mid', g)
    dec = _dec(sd)
    opts = dict(config.tiny_config().rendering_kwargs, depth_resolution=12, depth_resolution_importance=12)
    M = res * res
    try:
        for V in (1, 2):
            N = B * V
            _, _, cams, _ = weights.demo_inputs(config.tiny_config(), N, seed=6)
            u_c = torch.rand(N, M, 12, 1, generator=g)
            u_f = torch.rand(N * M, 12, generator=g)
            rgb, depth, wsum = torch.empty(N, M, 32, device=DEV), torch.empty(N, M, device=DEV), torch.empty(N, M, device=DEV)
            mm = torch.tensor([float('inf'), float('-inf')], device=DEV).expand(N, 2).contiguous()
            K.render_rays(planes, cams[:, :16].contiguous().to(DEV), cams[:, 16:25].contiguous().to(DEV), res, opts, dec, rgb, depth, wsum, mm,
                          u_coarse=u_c.to(DEV), u_fine=u_f.to(DEV), views=V, depth_range_per_image=1)
            K.depth_clamp_images(depth, mm)
            imgs = [i * V + v for i in check for v in range(V)]
            sel = torch.tensor(imgs)
            o, d = orr.ray_sampler(cams[sel, :16].reshape(-1, 4, 4), cams[sel, 16:25].reshape(-1, 3, 3), res)
            pl = host.repeat_interleave(V, 0)
            for j, n in enumerate(imgs):                        # per-image depth range: one oracle render per image
                r = orr.render(sd, pl[j:j + 1], o[j:j + 1], d[j:j + 1], opts, u_c[n:n + 1], u_f[n * M:(n + 1) * M])
                for name, x, y in (('rgb', rgb[n], r[0][0]), ('depth', depth[n], r[1][0, :, 0]), ('wsum', wsum[n], r[2][0, :, 0])):
                    e = range_rel_err(x.cpu(), y)
                    assert e < BOUNDS['oracle'], (V, n, name, e)
            del rgb, depth, wsum, mm
        # normals at N = 170
        N = B
        _, _, cams, _ = weights.demo_inputs(config.tiny_config(), N, seed=7)
        u_c = torch.rand(N, M, 12, 1, generator=g)
        u_f = torch.rand(N * M, 12, generator=g)
        rgb, depth, wsum = torch.empty(N, M, 32, device=DEV), torch.empty(N, M, device=DEV), torch.empty(N, M, device=DEV)
        mm = torch.tensor([float('inf'), float('-inf')], device=DEV)
        normal = torch.full((N, M, 3), float('nan'), device=DEV)
        work = torch.full((K.normals_workspace_floats(N, res, opts),), float('nan'), device=DEV)
        K.render_rays_normals(planes, cams[:, :16].contiguous().to(DEV), cams[:, 16:25].contiguous().to(DEV), res, opts, dec, rgb, depth, wsum,
                              mm, normal, work, u_coarse=u_c.to(DEV), u_fine=u_f.to(DEV))
        sel = torch.tensor(check)
        o, d = orr.ray_sampler(cams[sel, :16].reshape(-1, 4, 4), cams[sel, 16:25].reshape(-1, 3, 3), res)
        u_fs = u_f.view(N, M, 12)[sel].reshape(-1, 12)
        ref = onr.render_normals(sd, host, o, d, opts, u_c[sel], u_fs, return_samples=True)
        _check_against_oracle(sd, host, o, d, opts, work.view(N, M, -1)[sel.to(DEV)], normal[sel.to(DEV)], ref)
        del rgb, depth, wsum, mm, normal, work
        # sample_points at N = 170, a few points per set
        Pn = 40
        coords = (torch.rand(B, Pn, 3, generator=g) * 2 - 1) * 0.55
        sigma, prgb = torch.empty(B, Pn, device=DEV), torch.empty(B, Pn, 32, device=DEV)
        K.sample_points(planes, coords.to(DEV), 1.0, dec, sigma, prgb)
        rgb_ref, sig_ref = orr.run_model(sd, host, coords[sel], {'box_warp': 1.0})
        assert range_rel_err(sigma[sel.to(DEV)].cpu(), sig_ref[..., 0]) < BOUNDS['points']
        assert range_rel_err(prgb[sel.to(DEV)].cpu(), rgb_ref) < BOUNDS['points']
        del sigma, prgb
    finally:
        del planes
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ launched instances
@pytest.mark.gpu
def test_launched_kernels_match_plan(tmp_path):
    """Every case under torch.profiler: the render_fused_kernel<L, export> it launched (the template arguments are in the demangled
    name) and its grid are the ones `plan` predicts; normals_fused_kernel (not a template) and points_fused_kernel<rgb> likewise."""
    from next3d_b200 import kernels as K
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    setups = [setup_case(c) for c in CASES]
    devs = [_device_inputs(s) for s in setups]
    outs = [_outputs(c) for c in CASES]
    nouts = [(_outputs(c), torch.empty(c['N'], c['res'] ** 2, 3, device=DEV),
              torch.empty(K.normals_workspace_floats(c['N'], c['res'], s['opts']), device=DEV)) for c, s in zip(NORMAL_CASES, (setup_case(c) for c in NORMAL_CASES))]
    pts = [(pc, *_points_setup(pc)) for pc in POINT_CASES]
    torch.cuda.synchronize()

    def launch_all():
        """Every launch of the table; -> (case, kernel instance, grid) in launch order."""
        expected = []
        for s, dv, out in zip(setups, devs, outs):
            launch_case(s, out, dv)
            p = _plan(s['c'], sms)
            expected.append((s['c']['name'], f'render_fused_kernel<{p["L"]}, false>', p['grid']))
        for c, (out, normal, work) in zip(NORMAL_CASES, nouts):
            i = CASE_IDS.index(c['name'])
            launch_case(setups[i], out, devs[i], normal=normal, work=work)
            p = _plan(c, sms)
            expected.append((c['name'], f'render_fused_kernel<{p["L"]}, true>', p['grid']))
            expected.append((c['name'], 'normals_fused_kernel', normals_grid(c['N'], c['res'], sms)))
        for pc, planes, sd, coords in pts:
            launch_points(pc, planes, sd, coords)
            expected.append((pc['name'], f'points_fused_kernel<{"true" if pc["rgb"] else "false"}>', points_grid(*coords.shape[:2], sms)))
        return expected

    pat = re.compile(r'(render_fused_kernel<\d+, (?:true|false)>|normals_fused_kernel|points_fused_kernel<(?:true|false)>)')
    expected, events = launched_kernels(launch_all, pat, tmp_path)
    for (name, kernel, grid), e in zip(expected, events):
        assert pat.search(e['name']).group(1) == kernel, (name, e['name'], kernel)
        g = e.get('args', {}).get('grid')
        if g is not None:
            assert list(g) == [grid, 1, 1], (name, kernel, g, grid)


# ------------------------------------------------------------------------------------------------ alignment (CPU, nothing launched)
def _render_desc(planes_ptr):
    from next3d_b200 import config, kernels as K
    planes = torch.zeros(1, 3, 4, 4, 32)
    cam, intr = torch.zeros(1, 16), torch.zeros(1, 9)
    dec = (torch.zeros(64, 32), torch.zeros(64), torch.zeros(33, 64), torch.zeros(33))
    out = torch.zeros(4 * 4 * 32)
    p = K._render_full_desc(planes, cam, intr, 4, config.tiny_config().rendering_kwargs, dec, out, out, out, None, None, None, 0, None)
    p.planes = planes_ptr
    return p, out


@pytest.mark.parametrize('entry', ['n3d_render_rays', 'n3d_render_rays_normals'])
def test_render_refuses_misaligned_planes(entry):
    L = lib()
    buf = torch.zeros(3 * 4 * 4 * 32 + 64)
    p, out = _render_desc(offset_view(buf, 16).data_ptr())
    if entry == 'n3d_render_rays':
        rc = L.lib.n3d_render_rays(C.byref(p), None)
    else:
        rc = L.lib.n3d_render_rays_normals(C.byref(p), out.data_ptr(), out.data_ptr(), None)
    refused(rc, f'{entry}: planes must be 32-byte aligned')


def _sample_points(planes_ptr, rgb_ptr, N=1, PH=4, PW=4):
    L = lib()
    dec = [torch.zeros(n) for n in (64 * 32, 64, 33 * 64, 33)]
    coords, sigma = torch.zeros(N * 8 * 3), torch.zeros(N * 8)
    return L.lib.n3d_sample_points(planes_ptr, N, PH, PW, coords.data_ptr(), 8, 1.0, *(t.data_ptr() for t in dec), sigma.data_ptr(), rgb_ptr,
                                   None)


@pytest.mark.parametrize('field', ['planes', 'rgb'])
def test_sample_points_refuses_misaligned_buffers(field):
    planes = torch.zeros(3 * 4 * 4 * 32 + 64)
    rgb = torch.zeros(8 * 32 + 64)
    if field == 'planes':
        rc = _sample_points(offset_view(planes, 16).data_ptr(), rgb.data_ptr())
        refused(rc, 'n3d_sample_points: planes must be 32-byte aligned')
    else:
        rc = _sample_points(planes.data_ptr(), offset_view(rgb, 4).data_ptr())
        refused(rc, 'n3d_sample_points: rgb must be 8-byte aligned')


def test_sample_grid_refuses_misaligned_planes():
    L = lib()
    planes = torch.zeros(3 * 4 * 4 * 32 + 64)
    dec = [torch.zeros(n) for n in (64 * 32, 64, 33 * 64, 33)]
    grid = torch.zeros(8 ** 3)
    rc = L.lib.n3d_sample_grid(offset_view(planes, 16).data_ptr(), 4, 4, 8, C.c_float(1.0), C.c_float(1.0), 0, 8 ** 3, 0, C.c_float(-1000.0),
                               *(t.data_ptr() for t in dec), grid.data_ptr(), None)
    refused(rc, 'n3d_sample_grid: planes must be 32-byte aligned')
