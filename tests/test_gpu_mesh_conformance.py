"""The mesh and texture kernels of raster.cu against the oracle and fp64 references, over a table of launches that reaches every path
their entry points can take:

    n3d_transform_points  transform_kernel                          bit-exact vs oracle.generator._bmm3_fma + the view shift / scale
    n3d_rasterize         raster_setup_kernel + rasterize_kernel    bit-exact vs oracle.rasterize.rasterize_meshes (oracle_c.c)
    n3d_uv_sample         uv_sample_kernel                          fp64 F.grid_sample of the texture and of the eye mask
    n3d_fill_mouth        fill_mouth_kernel                         bit-exact vs oracle.generator.fill_mouth
    n3d_fill_mouth_binarize                                         the same, then the side-plane binarization of triplane_next3d.py:226
    n3d_mouth_box         mouth_box_kernel                          exact vs oracle.generator.gen_mouth_mask
    n3d_resize_aa         resize_aa_kernel / resize_aa_scalar_kernel   fp64 F.interpolate(bilinear, antialias=True), Python slicing
    n3d_blend_planes      blend_kernel                              fp64

Every output is a view into a larger allocation filled with a sentinel: the elements a launch owns must be written (and match), every
other element -- guard bands, destination pixels outside a paste box -- must keep the sentinel's bits.  Each case is then rerun and must
be bit-identical.  `plan` mirrors each entry point's launch rule in plain Python; the CPU test checks that the table covers everything
in COVERAGE, and the profiler test checks on the GPU that each case launched the kernels and grids the plan predicts.  The refusal
tests at the end need no GPU: arguments outside an entry point's contract must be refused before any device call.
"""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.helpers import Guarded, RangeErr, cdiv, grid_stride, launched_kernels, lib, record_errors, refused, rerun_identical

DEV = 'cuda'
SMS = 132                   # SM count the table is planned at (H100 SXM)

# Error bounds of the inexact kernels, each at most 4x the worst case measured over the table on an H100 80GB HBM3 (700 W power
# limit), which is given beside it.  uv: range-relative over the three texture planes, absolute on alpha (alpha lies in [0, 1]); both
# are dominated by the fp32 tap position ((u + 1) * W - 1) / 2, whose ulp at a 512-texel axis is 3e-5 of a texel.  resize:
# range-relative, fp32 output and hi + lo of the split output.  N3D_MESH_ERRORS=<file> appends every measured error to that file as
# JSON lines.
BOUNDS = {
    'uv.planes': 1e-4,      # Worst: 2.8e-5 (uv_c3_tex512)
    'uv.alpha': 1.9e-4,     # Worst: 4.9e-5 (uv_c31: 512x384 mask)
    'resize.f32': 1.4e-5,   # Worst: 3.6e-6 (rs_c32_paste64)
    'resize.split': 2e-5,   # Worst: 5.2e-6 (rs_c64; the split rounds at 2^-17 of the value)
    'blend': 4e-7,          # Worst: 1.0e-7 (bl_prod)
}


# ------------------------------------------------------------------------------------------------ the launch rules, mirrored
def resize_wide(C, aligned=True):
    """n3d_resize_aa: the warp-per-pixel kernel for C = 4 * 2^k <= 128 and a 16-byte aligned src, else one thread per element."""
    return C % 4 == 0 and C <= 128 and 32 % (C // 4) == 0 and aligned


def _aa_taps(out_i, in_size, out_size):
    """aa_axis (raster.cu): number of source taps of destination index out_i along one axis, in fp32 as the kernel has it."""
    f = np.float32
    scale = f(in_size) / f(out_size)
    support = scale if scale >= 1 else f(1)
    center = scale * (f(out_i) + f(0.5))
    lo = max(int(center - support + f(0.5)), 0)
    hi = min(int(center + support + f(0.5)), in_size)
    return hi - lo


def _windows(c):
    """Per image: (sy0, sx0, ih, iw, ty0, tx0, oh, ow) with the kernel's clipping (source box clipped to the image)."""
    out = []
    for n in range(c['N']):
        sy0, sy1, sx0, sx1 = c['src_box'][n] if c['src_box'] else (0, c['SH'], 0, c['SW'])
        ty0, ty1, tx0, tx1 = c['dst_box'][n] if c['dst_box'] else (0, c['DH'], 0, c['DW'])
        sy0, sx0, sy1, sx1 = max(sy0, 0), max(sx0, 0), min(sy1, c['SH']), min(sx1, c['SW'])
        out.append((sy0, sx0, sy1 - sy0, sx1 - sx0, ty0, tx0, ty1 - ty0, tx1 - tx0))
    return out


def resize_branches(c):
    """Inside resize_aa_kernel: 'all' (every lane a tap lane) where a pixel has >= 64 taps and C <= 32, else 'tap' (tap lanes x
    channel groups).  The set of branches the case's destination pixels take."""
    got = set()
    for sy0, sx0, ih, iw, ty0, tx0, oh, ow in _windows(c):
        ny = {_aa_taps(i, ih, oh) for i in range(oh)}
        nx = {_aa_taps(i, iw, ow) for i in range(ow)}
        for a in ny:
            for b in nx:
                got.add('all' if a * b >= 64 and c['C'] // 4 <= 8 else 'tap')
    return got


def plan(c, sms=SMS):
    """The kernels a case launches, in order, each as (name, grid)."""
    k = c['kind']
    if k == 'transform':
        return [('transform_kernel', (grid_stride(c['N'] * c['nviews'] * c['P'], sms, 8), 1, 1))]
    if k == 'raster':
        bins = cdiv(c['W'], 16) * cdiv(c['H'], 16)
        return [('raster_setup_kernel', (grid_stride(c['NM'] * c['F'], sms, 8), 1, 1)), ('rasterize_kernel', (bins, c['NM'], 1))]
    if k == 'uv':
        return [('uv_sample_kernel', (grid_stride(c['N'] * c['H'] * c['W'] * 32, sms, 16), 1, 1))]
    if k == 'fill':
        return [('fill_mouth_kernel', (c['NI'], 1, 1))]
    if k == 'box':
        return [('mouth_box_kernel', (cdiv(c['N'], 64), 1, 1))]
    if k == 'resize':
        pix = c['N'] * c['DH'] * c['DW']
        if resize_wide(c['C'], not c['misalign']):
            return [('resize_aa_kernel', (grid_stride(pix * 32 // 4, sms, 16), 1, 1))]
        return [('resize_aa_scalar_kernel', (grid_stride(pix * c['C'], sms, 16), 1, 1))]
    return [('blend_kernel', (grid_stride(c['N'] * 3 * c['H'] * c['W'] * 8, sms, 16), 1, 1))]


# ------------------------------------------------------------------------------------------------ the case table
def _tf(name, N, P, nviews, rot, zoff, flip, pts='random'):
    return dict(name=name, kind='transform', N=N, P=P, nviews=nviews, rot=rot, zoff=zoff, flip=flip, pts=pts)


def _ra(name, H, W, NM, mesh, F_):
    return dict(name=name, kind='raster', H=H, W=W, NM=NM, mesh=mesh, F=F_)


def _uv(name, N, H, W, C, TH, TW, MH, MW, mask):
    return dict(name=name, kind='uv', N=N, H=H, W=W, C=C, TH=TH, TW=TW, MH=MH, MW=MW, mask=mask)


def _fi(name, NI, H, W, masks, binarize=(0, 0)):
    return dict(name=name, kind='fill', NI=NI, H=H, W=W, masks=masks, binarize=binarize)


def _bx(name, N, lms):
    return dict(name=name, kind='box', N=N, lms=lms)


def _rs(name, N, SH, SW, C, DH, DW, src_box=None, dst_box=None, outs='dst', misalign=False):
    return dict(name=name, kind='resize', N=N, SH=SH, SW=SW, C=C, DH=DH, DW=DW, src_box=src_box, dst_box=dst_box, outs=outs,
                misalign=misalign)


def _bl(name, N, H, W):
    return dict(name=name, kind='blend', N=N, H=H, W=W)


DEMO_F = 9976
CASES = [
    # transform: the production calls (4 views, vertices with zoff 10 + NDC flip, landmarks plain), random rotations, P 1 .. 5091
    _tf('tf_views4_verts', 2, 5023, 4, 'views', 10.0, 1, pts='demo'),
    _tf('tf_views4_lms', 2, 68, 4, 'views', 0.0, 0, pts='lms'),
    _tf('tf_random_p1', 3, 1, 1, 'random', 0.0, 1, pts='zero'),
    _tf('tf_random_p68', 1, 68, 2, 'random', 10.0, 0),
    _tf('tf_random_p5091', 1, 5091, 3, 'random', 0.0, 0, pts='demo'),
    _tf('tf_views_grid', 16, 5091, 4, 'views', 10.0, 1, pts='demo'),
    # rasterize: the demo mesh, F around the 256-face chunk, special faces, every image size of the contract
    _ra('ra_demo_256', 256, 256, 4, 'demo', DEMO_F),
    _ra('ra_demo_250x130', 250, 130, 4, 'demo', DEMO_F),
    _ra('ra_f1_1x1', 1, 1, 2, 'single', 1),
    _ra('ra_f1_17x1', 17, 1, 1, 'single', 1),
    _ra('ra_f255_64', 64, 64, 2, 'mix', 255),
    _ra('ra_f256_64', 64, 64, 2, 'mix', 256),
    _ra('ra_f257_250x130', 250, 130, 2, 'mix', 257),
    _ra('ra_f600_nm8_64', 64, 64, 8, 'mix', 600),
    _ra('ra_f600_256', 256, 256, 2, 'mix', 600),
    _ra('ra_crowd_64', 64, 64, 2, 'crowd', 301),
    _ra('ra_centres_64', 64, 64, 2, 'centres', 98),
    # uv_sample: C < 32, texture and mask sizes other than the render size, non-uniform masks, taps beyond the atlas
    _uv('uv_c32_prod', 1, 256, 256, 32, 256, 256, 256, 256, 'ones'),
    _uv('uv_c1_tex128x96', 3, 64, 64, 1, 128, 96, 512, 384, 'random'),
    _uv('uv_c3_tex512', 1, 96, 80, 3, 512, 512, 256, 256, 'binary'),
    _uv('uv_c8', 3, 48, 40, 8, 64, 80, 256, 256, 'random'),
    _uv('uv_c31', 1, 128, 128, 31, 200, 120, 512, 384, 'binary'),
    _uv('uv_c32_small', 1, 8, 8, 32, 32, 32, 256, 256, 'random'),
    # fill_mouth: sizes, seeds, threshold values, the serpentine (many passes), the side-plane binarization
    _fi('fi_demo_256', 2, 256, 256, ['demo0', 'demo1'], binarize=(1, 2)),
    _fi('fi_walls_64_ni24', 24, 64, 64, ['walls'] * 24, binarize=(8, 16)),
    _fi('fi_walls_96x200', 3, 96, 200, ['walls'] * 3),
    _fi('fi_walls_1x300', 3, 1, 300, ['walls'] * 3),
    _fi('fi_walls_300x1', 3, 300, 1, ['walls'] * 3, binarize=(0, 3)),
    _fi('fi_walls_300x40', 2, 300, 40, ['walls'] * 2),
    _fi('fi_walls_40x300', 2, 40, 300, ['walls'] * 2, binarize=(1, 2)),
    _fi('fi_walls_512x396', 1, 512, 396, ['walls']),
    _fi('fi_serpentine_128', 1, 128, 128, ['serpentine']),
    _fi('fi_serpentine_256', 2, 256, 256, ['serpentine', 'walls']),
    # mouth_box
    _bx('bx_demo_n1', 1, 'demo'),
    _bx('bx_random_n65', 65, 'random'),
    _bx('bx_mixed_n130', 130, 'mixed'),
    # resize_aa: wide C 4 .. 128 (both branches for C <= 32), scalar C 1, 3, 12, 256, a misaligned src, boxes, outputs
    _rs('rs_c4_down', 2, 64, 64, 4, 8, 8, outs='both'),
    _rs('rs_c4_up', 1, 16, 12, 4, 40, 52),
    _rs('rs_c8_down_split', 2, 72, 60, 8, 9, 6, outs='split'),
    _rs('rs_c8_up', 3, 9, 11, 8, 30, 27, outs='both'),
    _rs('rs_c16_down', 1, 128, 128, 16, 12, 12, outs='split_nostyle'),
    _rs('rs_c16_mixed', 2, 20, 200, 16, 60, 30),
    _rs('rs_c32_crop', 2, 256, 256, 32, 64, 64, src_box=[[82, 122, 108, 148], [220, 262, 230, 270]]),
    _rs('rs_c32_paste64', 2, 64, 64, 32, 256, 256, dst_box=[[82, 122, 108, 148], [60, 113, 90, 143]]),
    _rs('rs_c32_paste256', 2, 256, 256, 32, 256, 256, dst_box=[[82, 122, 108, 148], [200, 240, 210, 250]]),
    _rs('rs_c32_sr64', 2, 64, 64, 32, 128, 128, outs='both'),
    _rs('rs_c32_sr256', 1, 256, 256, 32, 128, 128, outs='split'),
    _rs('rs_c32_identity', 1, 40, 56, 32, 40, 56),
    _rs('rs_c32_misaligned', 1, 50, 30, 32, 23, 61, misalign=True),
    _rs('rs_c64', 1, 48, 40, 64, 23, 61, outs='both'),
    _rs('rs_c128', 3, 32, 32, 128, 17, 9, outs='split'),
    _rs('rs_c1', 2, 50, 30, 1, 20, 70),
    _rs('rs_c3_sr64', 2, 64, 64, 3, 128, 128),
    _rs('rs_c3_sr256', 1, 256, 256, 3, 128, 128),
    _rs('rs_c12_paste', 2, 30, 30, 12, 64, 48, src_box=[[0, 30, 5, 40], [3, 25, 0, 30]], dst_box=[[10, 50, 4, 44], [0, 64, 0, 48]],
        outs='both'),
    _rs('rs_c256', 1, 24, 24, 256, 12, 13, outs='split'),
    # blend_planes
    _bl('bl_n3', 3, 40, 24),
    _bl('bl_grid', 1, 160, 192),
    _bl('bl_prod', 1, 256, 256),
]
CASE_IDS = [c['name'] for c in CASES]


def _of(kind, cs):
    return [(c, p) for c, p in cs if c['kind'] == kind]


def _resize_cover():
    items = {}
    for C in (4, 8, 16, 32):
        items[f'resize_aa wide C {C}: all-lanes and tap-lane branches'] = (
            lambda cs, C=C: set().union(*[resize_branches(c) for c, p in _of('resize', cs) if c['C'] == C and p[0][0] == 'resize_aa_kernel'])
            == {'all', 'tap'})
    return items


COVERAGE = {
    'transform: nviews 1, 2, 3, 4': lambda cs: {c['nviews'] for c, p in _of('transform', cs)} == {1, 2, 3, 4},
    'transform: zoff 0 and 10, ndc_flip 0 and 1': lambda cs: {(c['zoff'], c['flip']) for c, p in _of('transform', cs)} >= {(0.0, 0), (0.0, 1), (10.0, 0), (10.0, 1)},
    'transform: P 1, 68, 5023, 5091': lambda cs: {c['P'] for c, p in _of('transform', cs)} >= {1, 68, 5023, 5091},
    'transform: the VIEWS and random rotations': lambda cs: {c['rot'] for c, p in _of('transform', cs)} == {'views', 'random'},
    'transform: a grid-stride launch': lambda cs: any(c['N'] * c['nviews'] * c['P'] > p[0][1][0] * 256 for c, p in _of('transform', cs)),
    'rasterize: 256^2, 64^2, 250x130, 17x1, 1x1': lambda cs: {(c['H'], c['W']) for c, p in _of('raster', cs)} >= {(256, 256), (64, 64), (250, 130), (17, 1), (1, 1)},
    'rasterize: F 1, 255, 256, 257, ~600 and the demo mesh': lambda cs: {c['F'] for c, p in _of('raster', cs)} >= {1, 255, 256, 257, 600, DEMO_F},
    'rasterize: more than 256 faces in one bin': lambda cs: any(c['mesh'] == 'crowd' and c['F'] > 256 for c, p in _of('raster', cs)),
    'rasterize: duplicates across a chunk boundary': lambda cs: any(c['mesh'] == 'mix' and c['F'] > 256 for c, p in _of('raster', cs)),
    'rasterize: vertices and edges on pixel centres': lambda cs: any(c['mesh'] == 'centres' for c, p in _of('raster', cs)),
    'rasterize: NM 8': lambda cs: any(c['NM'] == 8 for c, p in _of('raster', cs)),
    'uv_sample: C 1, 3, 8, 31, 32': lambda cs: {c['C'] for c, p in _of('uv', cs)} >= {1, 3, 8, 31, 32},
    'uv_sample: textures of another size than the render': lambda cs: any((c['TH'], c['TW']) != (c['H'], c['W']) for c, p in _of('uv', cs)),
    'uv_sample: a 512^2 texture and a 128x96 texture': lambda cs: {(c['TH'], c['TW']) for c, p in _of('uv', cs)} >= {(512, 512), (128, 96)},
    'uv_sample: masks 256^2 and 512x384': lambda cs: {(c['MH'], c['MW']) for c, p in _of('uv', cs)} >= {(256, 256), (512, 384)},
    'uv_sample: non-uniform masks': lambda cs: {c['mask'] for c, p in _of('uv', cs)} >= {'random', 'binary', 'ones'},
    'uv_sample: N 1 and 3': lambda cs: {c['N'] for c, p in _of('uv', cs)} >= {1, 3},
    'uv_sample: grid-stride and sub-wave launches': lambda cs: {c['N'] * c['H'] * c['W'] * 32 > p[0][1][0] * 256 for c, p in _of('uv', cs)} == {False, True}
        and any(p[0][1][0] < SMS for c, p in _of('uv', cs)),
    'fill_mouth: 256^2, 64^2, 96x200, 1xW, Hx1, > 256 rows, > 256 columns, 512x396':
        lambda cs: {(c['H'], c['W']) for c, p in _of('fill', cs)} >= {(256, 256), (64, 64), (96, 200), (1, 300), (300, 1), (300, 40), (40, 300), (512, 396)},
    'fill_mouth: 512x396 is exactly 200 KB': lambda cs: any(c['H'] * (c['W'] + 4) == 200 * 1024 for c, p in _of('fill', cs)),
    'fill_mouth: NI 24': lambda cs: any(c['NI'] == 24 for c, p in _of('fill', cs)),
    'fill_mouth: the demo alpha and the serpentine at 128^2 and 256^2': lambda cs: {(m, c['H']) for c, p in _of('fill', cs) for m in c['masks']}
        >= {('demo0', 256), ('demo1', 256), ('serpentine', 128), ('serpentine', 256)},
    'fill_mouth: binarized and plain images in one launch': lambda cs: any(0 < c['binarize'][1] - c['binarize'][0] < c['NI'] for c, p in _of('fill', cs)),
    'mouth_box: N 1, 65, 130': lambda cs: {c['N'] for c, p in _of('box', cs)} >= {1, 65, 130},
    'resize_aa: wide C 4, 8, 16, 32, 64, 128': lambda cs: {c['C'] for c, p in _of('resize', cs) if p[0][0] == 'resize_aa_kernel'} == {4, 8, 16, 32, 64, 128},
    'resize_aa: scalar C 1, 3, 12, 256 and a misaligned C 32': lambda cs: {(c['C'], c['misalign']) for c, p in _of('resize', cs) if p[0][0] == 'resize_aa_scalar_kernel'}
        >= {(1, False), (3, False), (12, False), (256, False), (32, True)},
    **_resize_cover(),
    'resize_aa: up, down, mixed and identity': lambda cs: {(np.sign(c['DH'] - c['SH']), np.sign(c['DW'] - c['SW'])) for c, p in _of('resize', cs) if not c['src_box']}
        >= {(1, 1), (-1, -1), (1, -1), (0, 0)},
    'resize_aa: src box clipped at the bottom and right': lambda cs: any(c['src_box'] and any(b[1] > c['SH'] and b[3] > c['SW'] for b in c['src_box'])
                                                                       for c, p in _of('resize', cs)),
    'resize_aa: dst box pastes': lambda cs: any(c['dst_box'] for c, p in _of('resize', cs)),
    'resize_aa: outputs dst, hi/lo with and without style, both': lambda cs: {c['outs'] for c, p in _of('resize', cs)} == {'dst', 'split', 'split_nostyle', 'both'},
    'resize_aa: N*DH*DW not a multiple of 4': lambda cs: any(c['N'] * c['DH'] * c['DW'] % 4 for c, p in _of('resize', cs)),
    'resize_aa: SR 64 -> 128 and 256 -> 128 at C 32 and 3': lambda cs: {(c['SH'], c['C']) for c, p in _of('resize', cs) if c['DH'] == 128}
        >= {(64, 32), (256, 32), (64, 3), (256, 3)},
    'blend: N 3, H != W, a grid-stride launch': lambda cs: any(c['N'] == 3 and c['H'] != c['W'] for c, p in _of('blend', cs))
        and any(c['N'] * 3 * c['H'] * c['W'] * 8 > p[0][1][0] * 256 for c, p in _of('blend', cs)),
}


def test_case_table_covers_every_launch_path():
    """CPU: the table reaches everything listed in COVERAGE, according to the mirrored launch rules."""
    planned = [(c, plan(c)) for c in CASES]
    missing = [k for k, ok in COVERAGE.items() if not ok(planned)]
    assert not missing, missing
    assert len(set(CASE_IDS)) == len(CASE_IDS)


def _f32(x):
    return np.float32(x)


def _gen(c):
    return np.random.default_rng(3000 + CASE_IDS.index(c['name']))


def _tgen(c):
    return torch.Generator(device=DEV).manual_seed(3000 + CASE_IDS.index(c['name']))


def _demo():
    from next3d_b200 import weights
    m = weights.load_flame_demo()
    return m, weights.topology_buffers(m)


def _rotations(c, rng):
    from oracle import generator as og
    if c['rot'] == 'views':
        return torch.stack([og.angle2matrix(a) for a in og.VIEWS[:c['nviews']]])
    q = [np.linalg.qr(rng.standard_normal((3, 3)))[0] for _ in range(c['nviews'])]
    return torch.from_numpy(np.stack(q).astype(np.float32))


# ------------------------------------------------------------------------------------------------ meshes for the rasterizer
def _orient(tri, front=True):
    """tri [F,3,3]: order the vertices so that face_area = edge_fn(v0, v1, v2) is > 0 (front) or < 0 (back-facing)."""
    x, y = tri[..., 0].astype(np.float64), tri[..., 1].astype(np.float64)
    area = (x[:, 0] - x[:, 1]) * (y[:, 2] - y[:, 1]) - (y[:, 0] - y[:, 1]) * (x[:, 2] - x[:, 1])
    flip = (area < 0) if front else (area > 0)
    tri[flip] = tri[flip][:, [0, 2, 1]]
    return tri


def _random_tris(rng, n, span=1.3, zlo=0.3, zhi=5.0):
    c = rng.uniform(-span, span, (n, 1, 2))
    s = np.exp(rng.uniform(np.log(0.02), np.log(0.6), (n, 1, 1)))
    xy = np.clip(c + s * rng.standard_normal((n, 3, 2)), -7.9, 7.9)
    z = rng.uniform(zlo, zhi, (n, 3, 1))
    return _orient(np.concatenate([xy, z], -1).astype(np.float32))


def _special_tris(rng):
    """Faces every culling branch and edge case of the setup pass meets (front-facing unless noted)."""
    t = []
    t += [_orient(_random_tris(rng, 6, zlo=0.05, zhi=0.2), front=False)]                            # back-facing, in front
    tiny = np.array([[0.1, 0.1, 0.1], [0.1 + 5e-5, 0.1, 0.1], [0.1, 0.1 + 5e-5, 0.1]], np.float32)   # |area| 2.5e-9 <= 1e-8, not 0
    t += [_orient(tiny[None].copy()), _orient(tiny[None].copy(), front=False)]
    t += [_random_tris(rng, 4, span=0.5, zlo=-3.0, zhi=-0.1)]                                         # zmax < 0
    neg = _random_tris(rng, 4, span=0.5, zlo=0.1, zhi=0.3)
    neg[:, 0, 2] = -1.5                                                                               # some negative z: pz < 0 on part
    t += [neg]
    t += [np.array([[[-3.0, -3.0, 6.0], [3.0, -2.5, 6.0], [0.0, 3.5, 6.0]]], np.float32)]             # past NDC +-1 (background)
    t += [_orient(np.array([[[1.5, 1.5, 1.0], [3.0, 1.6, 1.0], [2.0, 3.0, 1.0]],
                            [[-7.9, -7.9, 1.0], [-2.0, -7.5, 1.0], [-6.0, -1.5, 1.0]]], np.float32))]  # wholly outside
    cop = _random_tris(rng, 6, span=0.4)
    cop[..., 2] = 0.25                                                                                # coplanar, overlapping
    t += [cop]
    return np.concatenate(t)


def build_mesh(c):
    """-> verts [NM, V, 3] fp32, faces [F, 3] int32 (every index < V)."""
    rng = _gen(c)
    NM, F_ = c['NM'], c['F']
    kind = c['mesh']
    if kind == 'demo':
        from oracle import generator as og
        m, topo = _demo()
        v = torch.from_numpy(m['verts'])[None]
        verts = []
        for view in og.VIEWS[:NM]:
            tv = og.transform_view(v, view)
            tv[:, :, 2] += 10
            tv[..., :2] = -tv[..., :2]
            verts.append(tv[0])
        return torch.stack(verts).contiguous(), topo['faces'][0][:, [0, 2, 1]].to(torch.int32).contiguous()
    if kind == 'single':
        tri = _orient(np.array([[[-0.9, -0.8, 1.0], [0.95, -0.2, 2.0], [-0.3, 0.9, 3.0]]], np.float32))
    elif kind == 'crowd':
        # 300 pixel-sized faces inside the 16x16 bin (bx 1, by 2) of a 64^2 image, in front of one large background face
        n = F_ - 1
        cxy = np.stack([rng.uniform(0.03, 0.47, n), rng.uniform(-0.47, -0.03, n)], -1)[:, None]
        xy = cxy + 0.03 * rng.standard_normal((n, 3, 2))
        tri = _orient(np.concatenate([xy, rng.uniform(0.5, 2.0, (n, 3, 1))], -1).astype(np.float32))
        tri = np.concatenate([np.array([[[-1.5, -1.5, 4.0], [1.5, -1.5, 4.0], [0.0, 1.5, 4.0]]], np.float32), tri])
    elif kind == 'centres':
        # 7x7 grid cells of 8x8 pixels with corners on pixel centres of a 64^2 image: every edge passes through pixel centres
        k = np.arange(4, 64, 8)
        p = (-1 + (2 * k + 1) / 64).astype(np.float32)
        tri = []
        for i in range(7):
            for j in range(7):
                a, b, cc, d = (p[i], p[j]), (p[i + 1], p[j]), (p[i + 1], p[j + 1]), (p[i], p[j + 1])
                z = np.float32(1 + (i + j) % 3)
                tri += [[(*a, z), (*b, z), (*cc, z)], [(*a, z), (*cc, z), (*d, z)]]
        tri = _orient(np.array(tri, np.float32))
    else:   # 'mix': special faces, then random ones up to F
        sp = _special_tris(rng)
        tri = np.concatenate([sp, _random_tris(rng, max(F_ - len(sp), 0))])[:F_]
    assert len(tri) == F_, (c['name'], len(tri))
    faces = np.arange(3 * F_, dtype=np.int32).reshape(F_, 3)
    if kind == 'mix':
        # coplanar duplicates: face g repeats face f's vertices, in the same order or rotated; inside one chunk and f, f + 256
        for f, g, rot in ((3, 40, 0), (7, 60, 1), (0, 256, 1), (2, 258, 0), (9, 265, 1)):
            if g < F_:
                faces[g] = np.roll(faces[f], rot)
                tri[f, :, 2] = np.float32(0.04)          # nearest of all, so the tie decides the pixel
    verts = np.repeat(tri.reshape(1, 3 * F_, 3), NM, 0)
    if NM > 1 and kind in ('mix', 'crowd'):
        verts[1:, :, :2] += (0.01 * rng.standard_normal((NM - 1, 3 * F_, 2))).astype(np.float32)   # other vertices per image
    return torch.from_numpy(np.ascontiguousarray(verts, np.float32)), torch.from_numpy(faces)


# ------------------------------------------------------------------------------------------------ fill_mouth inputs
def _edges(a0):
    """For seed value a0: the float32 alphas just inside and just outside [seed, seed + 254] on alpha * 255 (the kernel's and
    cv2's fixed range): (lo_in, lo_out, hi_in, hi_out); lo_out is None when it would be subnormal or negative zero."""
    seed = _f32(_f32(a0) * _f32(255))
    vmax = _f32(seed + _f32(254))
    prod = lambda a: _f32(_f32(a) * _f32(255))             # noqa: E731
    hi = _f32(vmax / 255)
    while prod(hi) > vmax:
        hi = np.nextafter(hi, _f32(-np.inf))
    while prod(np.nextafter(hi, _f32(np.inf))) <= vmax:
        hi = np.nextafter(hi, _f32(np.inf))
    lo = _f32(a0)
    while prod(np.nextafter(lo, _f32(-np.inf))) >= seed:
        lo = np.nextafter(lo, _f32(-np.inf))
    lo_out = np.nextafter(lo, _f32(-np.inf))
    return lo, (lo_out if a0 > 0 and prod(lo_out) < seed else None), hi, np.nextafter(hi, _f32(np.inf))


def _serpentine(n):
    """1-pixel staircase corridors (x - y) % 4 in {0, 1}, joined end to end into one 4-connected snake from the corner."""
    y, x = np.mgrid[0:n, 0:n]
    g = (((x - y) % 4) < 2).astype(np.float32)
    for k in range(-(n // 4) - 1, n // 4 + 1):
        a = 4 * k + 2
        for d in (a, a + 1):
            if k % 2 == 0:
                if 0 <= d < n:
                    g[0, d] = 1
                elif d < 0 and -d < n:
                    g[-d, 0] = 1
            else:
                if d >= 0 and n - 1 - d >= 0:
                    g[n - 1 - d, n - 1] = 1
                elif d < 0 and n - 1 + d >= 0:
                    g[n - 1, n - 1 + d] = 1
    return 1 - g           # fillable (alpha 0, the seed's value) along the snake, alpha 1 in the walls


def _walls(H, W, a0, rng):
    """Fillable values in [seed, seed + 254] (on alpha * 255) crossed by walls of values outside it: rectangle outlines (some clipped by
    the border), lines, and 1-pixel gates in them holding the values just inside / just outside the range."""
    lo_in, lo_out, hi_in, hi_out = _edges(a0)
    img = rng.uniform(a0, float(hi_in), (H, W)).astype(np.float32)
    wall = _f32(float(hi_out) + 0.25)
    gates = [v for v in (lo_in, lo_out, hi_in, hi_out) if v is not None]
    for _ in range(max(2, H * W // 400)):
        y0, x0 = rng.integers(-H // 4, H), rng.integers(-W // 4, W)
        y1, x1 = y0 + rng.integers(2, max(3, H // 2)), x0 + rng.integers(2, max(3, W // 2))
        ys, xs = slice(max(y0, 0), min(y1 + 1, H)), slice(max(x0, 0), min(x1 + 1, W))
        for yy in (y0, y1):
            if 0 <= yy < H:
                img[yy, xs] = wall
        for xx in (x0, x1):
            if 0 <= xx < W:
                img[ys, xx] = wall
        if 0 <= y0 < H and xs.stop - xs.start > 2:
            img[y0, rng.integers(xs.start + 1, xs.stop - 1)] = gates[rng.integers(len(gates))]
    if H > 8 and W > 8:
        img[H // 2, :] = np.where(rng.random(W) < 0.9, wall, img[H // 2, :])     # a leaky line across the image
    img[0, 0] = _f32(a0)
    return img


def _demo_alpha(view):
    """mask * visible of the demo mesh in one view, with a mask that is zero outside a face region (the side plane then has
    fractional values on the head outline)."""
    from oracle import generator as og
    m, topo = _demo()
    v = torch.from_numpy(m['verts'])[None]
    faces = topo['faces'][..., [0, 2, 1]]
    face_uv = topo['face_uvcoords'][:, :, [0, 2, 1]]
    tv = og.transform_view(v, og.VIEWS[view])
    tv[:, :, 2] += 10
    r, _ = og.rasterize_uv(tv, faces, face_uv)
    grid = r[:, :-1].permute(0, 2, 3, 1)[:, :, :, :2]
    return (F.grid_sample(face_region_mask(), grid, align_corners=False) * r[:, -1:])[0, 0].numpy()


def face_region_mask():
    """A binary 256^2 UV mask that is zero outside a face-shaped region."""
    m = torch.ones(1, 1, 256, 256)
    m[..., :, :40] = 0
    m[..., :, 216:] = 0
    m[..., 230:, :] = 0
    return m


def build_fill(c):
    rng = _gen(c)
    imgs = []
    for i, kind in enumerate(c['masks']):
        if kind.startswith('demo'):
            imgs.append(_demo_alpha(int(kind[-1])))
        elif kind == 'serpentine':
            imgs.append(_serpentine(c['H']))
        else:
            imgs.append(_walls(c['H'], c['W'], (0.0, 0.5, 1.0)[i % 3], rng))
    return torch.from_numpy(np.stack(imgs).astype(np.float32))


def fill_reference(alpha, binarize):
    from oracle import generator as og
    ref = og.fill_mouth(alpha[:, None].clone())[:, 0]
    b0, b1 = binarize
    ref[b0:b1] = (ref[b0:b1].bool() | ref[b0:b1].bool()).float()        # the side plane as triplane_next3d.py:226 has it
    return ref


# ------------------------------------------------------------------------------------------------ mouth_box inputs
def _near_integer_extents():
    """Extents (multiples of 1/8, exact after lm * 128 + 128) whose fp32 ext * 1.2 lies within 4 ulps of an integer."""
    out = []
    for k in range(16, 960):
        e = _f32(k / 8)
        p = _f32(e * _f32(1.2))
        if p != np.round(p) and abs(p - np.round(p)) <= 4 * np.spacing(p):
            out.append(e)
    return out


def build_landmarks(c):
    rng = _gen(c)
    N = c['N']
    from oracle import generator as og
    m, _ = _demo()
    demo = og.transform_view(torch.from_numpy(m['lms'])[None], og.VIEWS[0])[0, :, :2].numpy()
    out = []
    kinds = {'demo': ['demo'], 'random': ['random'], 'mixed': ['demo', 'random', 'negative', 'near_int']}[c['lms']]
    near = _near_integer_extents()
    assert len(near) >= 8, near
    for n in range(N):
        kind = kinds[n % len(kinds)]
        if kind == 'demo':
            lm = demo + 0.01 * rng.standard_normal(demo.shape)
        elif kind == 'random':
            lm = rng.uniform(-0.9, 0.9, (68, 2))
        elif kind == 'negative':             # mouth at the top-left corner: avg - side // 2 < 0 (truncation toward zero)
            lm = rng.uniform(-1.0, -0.85, (68, 2))
            lm[48:60] = rng.uniform(-0.999, -0.7, (12, 2))
        else:                                # extents where ext * 1.2 lands next to an integer
            lm = rng.uniform(-0.5, 0.5, (68, 2))
            e = near[n % len(near)]
            base = np.round(rng.uniform(-0.3, 0.1, 2) * 1024) / 1024
            q = np.round(rng.uniform(0, 1, (12, 2)) * float(e) * 8) / 1024           # inside the extent, on the 1/1024 grid
            lm[48:60] = base + np.minimum(q, float(e) / 128)
            lm[48, 0], lm[54, 0] = base[0], base[0] + float(e) / 128                 # x spans exactly e (after * 128)
            lm[48:60, 1] = base[1] + np.minimum(q[:, 1], float(e) / 256)             # y spans less
        out.append(lm)
    return torch.from_numpy(np.stack(out).astype(np.float32))


# ------------------------------------------------------------------------------------------------ setup and launch
def _rnd(g, *shape):
    return torch.randn(*shape, device=DEV, generator=g)


def setup_case(c):
    """Inputs and guarded outputs of a case (the device tensors every launch points at)."""
    k = c['kind']
    g = _tgen(c)
    s = dict(c=c, outs={})
    if k == 'transform':
        rng = _gen(c)
        if c['pts'] in ('demo', 'lms'):
            m, _ = _demo()
            p = {5023: m['verts'], 68: m['lms'], 5091: np.concatenate([m['verts'], m['lms']])}[c['P']]
            jitter = 1e-3 * rng.standard_normal((c['N'], c['P'], 3)) * (np.arange(c['N']) > 0)[:, None, None]    # image 0: the mesh itself
            p = np.repeat(p[None], c['N'], 0) + jitter
        elif c['pts'] == 'zero':
            p = np.zeros((c['N'], c['P'], 3))
            p[1:] = rng.standard_normal((c['N'] - 1, c['P'], 3)) * 0.1
        else:
            p = rng.standard_normal((c['N'], c['P'], 3)) * 0.1
        s['pts'] = torch.from_numpy(p.astype(np.float32))
        s['rot'] = _rotations(c, rng)
        s['pts_d'], s['rot_d'] = s['pts'].to(DEV), s['rot'].to(DEV)
        s['outs']['out'] = Guarded((c['N'], c['nviews'], c['P'], 3), torch.float32)
    elif k == 'raster':
        verts, faces = build_mesh(c)
        s['verts'], s['faces'] = verts, faces
        s['verts_d'], s['faces_d'] = verts.to(DEV), faces.to(DEV)
        NM, H, W = c['NM'], c['H'], c['W']
        s['outs'] = dict(p2f=Guarded((NM, H, W), torch.int32), bary=Guarded((NM, H, W, 3), torch.float32),
                         ws=Guarded((NM * c['F'] * 16,), torch.float32))
    elif k == 'uv':
        N, H, W, C = c['N'], c['H'], c['W'], c['C']
        F_ = 500
        p2f = torch.randint(0, F_, (N * 4, H, W), device=DEV, generator=g, dtype=torch.int32)
        p2f[torch.rand(N * 4, H, W, device=DEV, generator=g) < 0.25] = -1                              # background pixels
        b = torch.rand(N * 4, H, W, 3, device=DEV, generator=g) + 0.02
        b = (b / b.sum(-1, keepdim=True)).float()
        b[p2f < 0] = -1.0
        s['p2f'], s['bary'] = p2f, b.contiguous()
        s['face_uv'] = (torch.rand(F_, 3, 2, device=DEV, generator=g) * 2.4 - 1.2).contiguous()        # taps beyond the atlas
        s['tex'] = _rnd(g, N, c['TH'], c['TW'], C)
        MH, MW = c['MH'], c['MW']
        mask = {'ones': torch.ones(MH, MW, device=DEV), 'random': torch.rand(MH, MW, device=DEV, generator=g),
                'binary': (torch.rand(MH // 16, MW // 16, device=DEV, generator=g) < 0.6).float().repeat_interleave(16, 0).repeat_interleave(16, 1)}
        s['mask'] = mask[c['mask']].contiguous()
        s['outs'] = dict(planes=Guarded((3, N, H, W, C), torch.float32), alpha=Guarded((3, N, H, W), torch.float32))
    elif k == 'fill':
        s['alpha_in'] = build_fill(c)
        s['outs']['alpha'] = Guarded(tuple(s['alpha_in'].shape), torch.float32)
    elif k == 'box':
        s['lm'] = build_landmarks(c)
        s['lm_d'] = s['lm'].to(DEV)
        s['outs']['boxes'] = Guarded((c['N'], 4), torch.int32)
    elif k == 'resize':
        N, SH, SW, C, DH, DW = c['N'], c['SH'], c['SW'], c['C'], c['DH'], c['DW']
        n = N * SH * SW * C
        flat = _rnd(g, n + 4)
        s['src'] = (flat[1:n + 1] if c['misalign'] else flat[:n]).view(N, SH, SW, C)
        s['src_box'] = torch.tensor(c['src_box'], dtype=torch.int32, device=DEV) if c['src_box'] else None
        s['dst_box'] = torch.tensor(c['dst_box'], dtype=torch.int32, device=DEV) if c['dst_box'] else None
        own = None
        if c['dst_box']:
            own = torch.zeros(N, DH, DW, 1, dtype=torch.bool, device=DEV)
            for i, (y0, y1, x0, x1) in enumerate(c['dst_box']):
                own[i, y0:y1, x0:x1] = True
        s['style'] = _rnd(g, N, C) if c['outs'] in ('split', 'both') else None
        if c['outs'] in ('dst', 'both'):
            s['outs']['dst'] = Guarded((N, DH, DW, C), torch.float32, own)
        if c['outs'] != 'dst':
            s['outs']['hi'] = Guarded((N, DH, DW, C), torch.bfloat16, own)
            s['outs']['lo'] = Guarded((N, DH, DW, C), torch.bfloat16, own)
    else:
        N, H, W = c['N'], c['H'], c['W']
        s['front'], s['tex'], s['stat'] = _rnd(g, N, H, W, 32), _rnd(g, 3, N, H, W, 32), _rnd(g, N, H, W, 96)
        a = torch.rand(3, N, H, W, device=DEV, generator=g)
        r = torch.rand(3, N, H, W, device=DEV, generator=g)
        a[r < 0.2] = 0.0
        a[r > 0.8] = 1.0                                                                                # alpha exactly 0 and 1
        s['alpha'] = a
        s['outs']['planes'] = Guarded((N, 3, H, W, 32), torch.float32)
    return s


def launch_case(s):
    from next3d_b200 import kernels as K
    c, o = s['c'], s['outs']
    k = c['kind']
    if k == 'transform':
        K.transform_points(s['pts_d'], s['rot_d'], c['zoff'], bool(c['flip']), o['out'].view)
    elif k == 'raster':
        K.rasterize(s['verts_d'], s['faces_d'], c['H'], c['W'], o['p2f'].view, o['bary'].view, workspace=o['ws'].view)
    elif k == 'uv':
        K.uv_sample(s['p2f'], s['bary'], s['face_uv'], s['tex'], s['mask'], o['planes'].view, o['alpha'].view)
    elif k == 'fill':
        o['alpha'].view.copy_(s['alpha_in'])
        if c['binarize'] != (0, 0):
            K.fill_mouth(o['alpha'].view, binarize=c['binarize'])
        else:
            K.fill_mouth(o['alpha'].view)
    elif k == 'box':
        K.mouth_box(s['lm_d'], o['boxes'].view)
    elif k == 'resize':
        d, hi, lo = (o[n].view if n in o else None for n in ('dst', 'hi', 'lo'))
        K.resize_aa(s['src'], d, c['DH'], c['DW'], src_box=s['src_box'], dst_box=s['dst_box'], style=s['style'], hi=hi, lo=lo)
    else:
        K.blend_planes(s['front'], s['tex'], s['alpha'], s['stat'], o['planes'].view)


# ------------------------------------------------------------------------------------------------ references and checks
def transform_reference(pts, rot, zoff, flip):
    """oracle.transform_view with the view's R, then z + zoff and the optional NDC flip, all in fp32 as the oracle has them (the camera
    add of +0 on x and y turns a -0 into +0 before y is negated, exactly as in transform_view)."""
    from oracle import generator as og
    N = pts.shape[0]
    out = []
    p = pts.clone()
    p[..., 1] *= -1
    for R in rot:
        r = og._bmm3_fma(p, R[None].expand(N, -1, -1))
        x = (r[..., 0] + 0.0) * 5.0 + 0.0
        y = -((r[..., 1] + torch.tensor(-0.01)) * 5.0 + 0.0)
        z = -((r[..., 2] + torch.tensor(-0.01)) * 5.0) + torch.tensor(zoff, dtype=torch.float32)
        if flip:
            x, y = -x, -y
        out.append(torch.stack([x, y, z], -1))
    return torch.stack(out, 1)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _mismatch(got, ref):
    """Count and first index of bitwise differences between two fp32 / int32 tensors."""
    d = _bits(got.cpu()) != _bits(ref.cpu())
    return int(d.sum()), (d.nonzero()[0].tolist() if d.any() else None)


def uv_reference(s):
    """fp64: u, v = sum_k bary_k * face_uv[f, k] (0, 0 on background); F.grid_sample (bilinear, zeros, align_corners False) of the
    texture and the mask; planes (view 0, view 1 + view 2, view 3); alpha = mask * visible of views 0, 1, 3."""
    c = s['c']
    N = c['N']
    p2f, bary = s['p2f'].long(), s['bary'].double()
    fu = s['face_uv'].double()[p2f.clamp_min(0)]                        # [N*4, H, W, 3, 2]
    uv = (bary[..., None] * fu).sum(-2)
    vis = (p2f >= 0)
    uv[~vis] = 0.0
    uv = uv.view(N, 4, c['H'], c['W'], 2)
    vis = vis.view(N, 4, c['H'], c['W']).double()
    tex = s['tex'].permute(0, 3, 1, 2).double()
    mask = s['mask'].double()[None, None].expand(N, -1, -1, -1)
    gs = lambda img, v: F.grid_sample(img, uv[:, v], mode='bilinear', padding_mode='zeros', align_corners=False)   # noqa: E731
    planes = [gs(tex, 0), gs(tex, 1) + gs(tex, 2), gs(tex, 3)]
    alpha = [gs(mask, v)[:, 0] * vis[:, v] for v in (0, 1, 3)]
    return [p.permute(0, 2, 3, 1) for p in planes], alpha


def resize_reference(s, n):
    """Image n's destination window and its fp64 value [oh, ow, C] (F.interpolate of the clipped source crop)."""
    c = s['c']
    sy0, sx0, ih, iw, ty0, tx0, oh, ow = _windows(c)[n]
    crop = s['src'][n, sy0:sy0 + ih, sx0:sx0 + iw].permute(2, 0, 1).double().cpu()[None]
    r = F.interpolate(crop, size=(oh, ow), mode='bilinear', align_corners=False, antialias=True)[0].permute(1, 2, 0)
    return (slice(ty0, ty0 + oh), slice(tx0, tx0 + ow)), r.to(DEV)


def check_case(s):
    """-> {bound kind: error} of the inexact kernels; asserts the bit-exact comparisons and the sentinel / written checks first."""
    c, o = s['c'], s['outs']
    k = c['kind']
    for name, t in o.items():
        assert t.untouched_ok(), f'{c["name"]}: an element outside `{name}` was written'
        assert t.written(), f'{c["name"]}: an element of `{name}` was not written'
    errs = {}
    if k == 'transform':
        ref = transform_reference(s['pts'], s['rot'], c['zoff'], c['flip'])
        n, where = _mismatch(o['out'].view, ref)
        assert n == 0, f'{c["name"]}: {n} values differ from the oracle (first at {where})'
    elif k == 'raster':
        from oracle import rasterize as orast
        NM, F_ = c['NM'], c['F']
        p2f, _, bary = orast.rasterize_meshes(s['verts'].numpy(), s['faces'][None].expand(NM, -1, -1).numpy(), c['H'], c['W'])
        p2f = p2f - (np.arange(NM)[:, None, None] * F_) * (p2f >= 0)
        n, where = _mismatch(o['p2f'].view, torch.from_numpy(p2f.astype(np.int32)))
        assert n == 0, f'{c["name"]}: pix_to_face differs from the oracle at {n} pixels (first at {where})'
        n, where = _mismatch(o['bary'].view, torch.from_numpy(bary))
        assert n == 0, f'{c["name"]}: barycentrics differ from the oracle at {n} values (first at {where})'
    elif k == 'uv':
        planes, alpha = uv_reference(s)
        e = RangeErr()
        for p in range(3):
            e.add(o['planes'].view[p], planes[p])
        errs['uv.planes'] = e.value()
        errs['uv.alpha'] = max((o['alpha'].view[p].double() - alpha[p]).abs().max().item() for p in range(3))
    elif k == 'fill':
        ref = fill_reference(s['alpha_in'], c['binarize'])
        n, where = _mismatch(o['alpha'].view, ref)
        assert n == 0, f'{c["name"]}: {n} alpha values differ from the oracle (first at {where})'
    elif k == 'box':
        from oracle import generator as og
        ref = og.gen_mouth_mask(s['lm'])
        got = o['boxes'].view.cpu().numpy()
        assert np.array_equal(got, ref), (c['name'], np.argwhere(got != ref)[:4].tolist())
    elif k == 'resize':
        e32, esp = RangeErr(), RangeErr()
        for n in range(c['N']):
            (ys, xs), ref = resize_reference(s, n)
            if 'dst' in o:
                e32.add(o['dst'].view[n, ys, xs], ref)
            if 'hi' in o:
                r = ref * s['style'][n].double() if s['style'] is not None else ref
                esp.add(o['hi'].view[n, ys, xs].double() + o['lo'].view[n, ys, xs].double(), r)
        if 'dst' in o:
            errs['resize.f32'] = e32.value()
        if 'hi' in o:
            errs['resize.split'] = esp.value()
    else:
        a = s['alpha'].double()
        tex = torch.cat([s['front'][None], s['tex'][1:]]).double()                   # [3, N, H, W, 32]
        stat = s['stat'].double().view(c['N'], c['H'], c['W'], 3, 32).permute(3, 0, 1, 2, 4)
        ref = (tex * a[..., None] + stat * (1 - a[..., None])).permute(1, 0, 2, 3, 4)
        e = RangeErr()
        e.add(o['planes'].view, ref)
        errs['blend'] = e.value()
        exact = ((a == 0) | (a == 1)).permute(1, 0, 2, 3)
        sel = torch.where((a == 1)[..., None], tex, stat).permute(1, 0, 2, 3, 4)
        assert torch.equal(o['planes'].view[exact].double(), sel[exact]), f'{c["name"]}: alpha 0 / 1 does not select exactly'
    return errs


@pytest.mark.gpu
@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_kernel_matches_reference(c):
    s = setup_case(c)
    launch_case(s)
    torch.cuda.synchronize()
    errs = check_case(s)
    record_errors('N3D_MESH_ERRORS', [{'case': c['name'], 'kind': k, 'err': e, 'bound': BOUNDS[k]} for k, e in errs.items()])
    bad = {k: e for k, e in errs.items() if not e < BOUNDS[k]}
    assert not bad, bad
    assert rerun_identical(list(s['outs'].values()), lambda: launch_case(s)), f'{c["name"]}: a rerun is not bit-identical'


@pytest.mark.gpu
def test_launched_kernels_match_plan(tmp_path):
    """Every case under torch.profiler: the kernels it launched and their grids are the ones `plan` predicts at the device's SM
    count."""
    names = ('raster_setup_kernel', 'rasterize_kernel', 'transform_kernel', 'uv_sample_kernel', 'fill_mouth_kernel', 'mouth_box_kernel',
             'resize_aa_scalar_kernel', 'resize_aa_kernel', 'blend_kernel')
    pattern = re.compile(r'(?<![\w])(' + '|'.join(names) + r')(?![\w])')
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    setups = [setup_case(c) for c in CASES]
    torch.cuda.synchronize()

    def run():
        expected = []
        for s in setups:
            launch_case(s)
            torch.cuda.synchronize()
            expected += [(s['c']['name'], kernel, grid) for kernel, grid in plan(s['c'], sms)]
        return expected

    expected, events = launched_kernels(run, pattern, tmp_path)
    for (who, kernel, grid), e in zip(expected, events):
        assert pattern.search(e['name']).group(1) == kernel, (who, e['name'], kernel)
        got = e.get('args', {}).get('grid')
        if got is not None:
            assert tuple(got) == grid, (who, kernel, got, grid)


# ------------------------------------------------------------------------------------------------ the engine's alpha under a face mask
@pytest.mark.gpu
def test_engine_alpha_matches_oracle_under_face_mask():
    """compute_planes with a UV mask that is zero outside a face region: the side plane's alpha has fractional values on the head
    outline before the reference binarizes it (triplane_next3d.py:226).  All three alpha planes must match the oracle's."""
    from next3d_b200 import config, weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    from oracle import generator as og
    cfg = config.tiny_config(512)
    sd = weights.make_state_dict(cfg, seed=3)
    G = TriPlaneGenerator.from_config(cfg, sd, device=DEV)
    G.uv_face_mask = face_region_mask()
    z, c_cond, _, v = weights.demo_inputs(cfg, 2, seed=3)
    with torch.no_grad():
        ws = G.mapping(z.to(DEV), c_cond.to(DEV), truncation_psi=0.7, truncation_cutoff=14)
        _, inter = G._get_engine().compute_planes(ws, v.to(DEV), return_intermediates=True)
    torch.cuda.synchronize()
    got = inter['alpha'].cpu()                                              # [3, N, H, W]: views 0, 1 (side), 3
    _, alphas, _, _ = og.rasterize(sd, v[:, :5023], v[:, 5023:], torch.zeros(2, 32, 256, 256), face_region_mask())
    side = alphas[1][:, 0]
    for p in (0, 2):
        assert (got[p] - alphas[p][:, 0]).abs().max().item() < 1e-6, p
    flips = (got[1] != side).nonzero().tolist()
    assert not flips, f'side-plane alpha differs from the oracle at {len(flips)} pixels, e.g. {flips[:8]}'
    assert set(got[1].unique().tolist()) <= {0.0, 1.0}


# ------------------------------------------------------------------------------------------------ CPU: the oracle, refusals
def test_oracle_flood_fill_fills_the_whole_serpentine():
    """CPU: oracle.generator.fill_mouth (oracle_c.c's flood fill) reaches every pixel of the serpentine 4-connected to the corner."""
    from scipy import ndimage
    from oracle import generator as og
    for n in (128, 256):
        a = torch.from_numpy(_serpentine(n))
        lab, _ = ndimage.label(a.numpy() == 0)                              # default structure: 4-connectivity
        reach = lab == lab[0, 0]
        assert reach.sum() > n * n // 3
        out = og.fill_mouth(a[None, None])[0, 0].numpy()
        # reached pixels: alpha 0 + 0 (filled: m = 1) -> 0; unreached fillable would be 0 + 1 -> 1; walls stay 1
        assert np.array_equal(out == 0, reach), n


def test_fill_edges_are_exact():
    """CPU: the threshold alphas the fill cases use sit exactly at the edges of [seed, seed + 254] on alpha * 255."""
    for a0 in (0.0, 0.5, 1.0):
        lo_in, lo_out, hi_in, hi_out = _edges(a0)
        seed = _f32(_f32(a0) * _f32(255))
        vmax = _f32(seed + _f32(254))
        prod = lambda a: _f32(_f32(a) * _f32(255))         # noqa: E731
        assert seed <= prod(lo_in) <= vmax and seed <= prod(hi_in) <= vmax
        assert prod(hi_out) > vmax and np.nextafter(hi_in, _f32(np.inf)) == hi_out
        assert lo_out is None or prod(lo_out) < seed


def test_uv_sample_refuses_more_than_32_channels():
    L = lib()
    t = torch.zeros(1024)
    p = t.data_ptr()
    refused(L.lib.n3d_uv_sample(p, p, p, p, p, 1, 4, 4, 4, 4, 33, 4, 4, p, p, None), 'C 33 > 32')


@pytest.mark.parametrize('what', ['images', 'workspace'])
def test_rasterize_refuses_bad_launches(what):
    L = lib()
    t = torch.zeros(4096)
    p = t.data_ptr()
    if what == 'images':
        refused(L.lib.n3d_rasterize(p, p, 65536, 3, 1, 16, 16, p, p, p, None), 'too many images (65536)')
    else:
        assert p % 16 == 0
        refused(L.lib.n3d_rasterize(p, p, 1, 3, 1, 16, 16, p, p, p + 4, None), 'workspace must be 16-byte aligned')


@pytest.mark.parametrize('H,W,b0,b1,what', [(512, 397, 0, 0, 'too large'), (397, 512, 0, 1, 'too large'), (8, 8, 0, 3, 'binarized images'),
                                             (8, 8, 1, 0, 'binarized images'), (8, 8, -1, 1, 'binarized images')])
def test_fill_mouth_refuses_bad_launches(H, W, b0, b1, what):
    L = lib()
    t = torch.zeros(16)
    refused(L.lib.n3d_fill_mouth_binarize(t.data_ptr(), 2, H, W, b0, b1, None), what)
    if what == 'too large':
        refused(L.lib.n3d_fill_mouth(t.data_ptr(), 2, H, W, None), what)


def test_resize_aa_refuses_hi_without_lo():
    L = lib()
    t = torch.zeros(1024)
    p = t.data_ptr()
    refused(L.lib.n3d_resize_aa(p, 1, 4, 4, 4, None, None, 4, 4, None, None, p, None, None), 'hi without lo')
