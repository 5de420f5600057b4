"""Thin torch-tensor wrappers over the C ABI (one Python function per extern "C" entry point of the engine).

Tensors are only used as owners of device memory; every call passes raw pointers + sizes and the current CUDA
stream.  Layout conventions: activations NHWC fp32 or split bf16 (hi, lo); weights packed [T, Cout, Cin] split bf16.  The opt-in
fp16 super-resolution head uses fp16 single tensors instead of the split pairs (the `f16` arguments).
"""
import ctypes as C

import torch

from . import _lib
from ._lib import lib, check, ptr, stream_ptr

BF16 = torch.bfloat16

# Kernels launched through this module so far (Engine.launches is its difference across one forward).  One counter per process is
# enough: the supported multi-GPU model is one process per GPU (DESIGN.md section 7).
launches = 0


def _run(fn, *args, kernels=1):
    """Call entry point `fn`, raise on an error status, and count the `kernels` it launches."""
    global launches
    check(getattr(lib, fn)(*args), fn)
    launches += kernels


# ------------------------------------------------------------------------------------------------ packing helpers
def split_bf16(x):
    """fp32 tensor -> (hi, lo) bf16 with hi + lo ~= x (host/torch-side, used for one-time weight packing)."""
    hi = x.to(BF16)
    lo = (x - hi.to(torch.float32)).to(BF16)
    return hi, lo


def pack_conv_weight(w, gain=1.0):
    """[Cout, Cin, kh, kw] fp32 -> split bf16 [kh*kw, Cout, Cin] (tap-major, tap = ky*kw + kx), pre-multiplied by `gain`."""
    cout, cin, kh, kw = w.shape
    wp = (w.to(torch.float32) * gain).permute(2, 3, 0, 1).reshape(kh * kw, cout, cin).contiguous()
    return split_bf16(wp)


def taps_conv3x3():
    return [(ky - 1, kx - 1, 0, ky * 3 + kx) for ky in range(3) for kx in range(3)]


def taps_conv1x1():
    return [(0, 0, 0, 0)]


def taps_transposed(a, b):
    """Stride-2 transposed 3x3 conv, output parity class (a, b): out[2p+a, 2q+b] += W[ky,kx] * x[p-(ky-a)/2, q-(kx-b)/2]."""
    return [(-(ky - a) // 2, -(kx - b) // 2, 0, ky * 3 + kx) for ky in range(3) for kx in range(3)
            if (ky - a) % 2 == 0 and (kx - b) % 2 == 0]


def taps_stride2():
    """Stride-2 3x3 conv over parity-split sub-images: F[2p+ky, 2q+kx] = sub[(ky&1)*2 + (kx&1)][p + ky//2, q + kx//2]."""
    return [(ky >> 1, kx >> 1, (ky & 1) * 2 + (kx & 1), ky * 3 + kx) for ky in range(3) for kx in range(3)]


def pack_conv_weight_f16(w, gain=1.0):
    """[Cout, Cin, kh, kw] fp32 -> fp16 [kh*kw, Cout, Cin] (tap-major), pre-multiplied by `gain` ([Cout] or a scalar) before the rounding."""
    cout, cin, kh, kw = w.shape
    g = torch.as_tensor(gain, dtype=torch.float32, device=w.device).reshape(-1, 1, 1, 1)
    return (w.to(torch.float32) * g).permute(2, 3, 0, 1).reshape(kh * kw, cout, cin).to(torch.float16).contiguous()


def make_split_out(hi=None, lo=None, style=None, cstride=0, coff=0, f16=False):
    """Output descriptor: split bf16 (hi, lo), or with f16 one fp16 tensor `hi` (lo unused)."""
    return _lib.SplitOut(ptr(hi), ptr(lo), ptr(style), cstride, coff, int(f16))


# ------------------------------------------------------------------------------------------------ kernels
def _conv_desc(a_hi, a_lo, w_hi, w_lo, N, MH, MW, nprod):
    """ConvGemm descriptor with the operands (a_*: bf16 [NI, AH, AW, Cin]; w_*: bf16 [T, Cout, Cin]; or, fp16 single operands, a_hi fp16
    and w_hi fp16 with a_lo = w_lo = None and nprod 1) and the M-space filled in."""
    NI, AH, AW, Cin = a_hi.shape
    T, Cout, Cin_w = w_hi.shape
    assert Cin_w == Cin, (Cin_w, Cin)
    p = _lib.ConvGemm()
    p.a_hi, p.a_lo = ptr(a_hi), ptr(a_lo)
    p.NI, p.AH, p.AW, p.Cin = NI, AH, AW, Cin
    p.w_hi, p.w_lo = ptr(w_hi), ptr(w_lo)
    p.T, p.Cout = T, Cout
    p.N, p.MH, p.MW = N, MH, MW
    p.nprod = nprod
    p.f16 = int(a_hi.dtype == torch.float16)
    if p.f16 and (w_hi.dtype != torch.float16 or a_lo is not None or w_lo is not None or nprod != 1):
        raise ValueError('conv_gemm: fp16 operands are one fp16 activation and one fp16 weight tensor, nprod 1')
    return p


def conv_gemm(a_hi, a_lo, w_hi, w_lo, taps, N, MH, MW, *, a_img_mul=0, nprod=3, mode=0, dcoef=None, bias=None, noise=None,
              noise_nstride=0, gain=1.0, slope=1.0, clamp=-1.0, outs=(), out_f32=None, f32_cstride=0, f32_coff=0, f32_nchw=False,
              f32_accumulate=False, oy_mul=1, oy_off=0, ox_mul=1, ox_off=0, OH=None, OW=None, rgb=None, splits=1, split_stride=0):
    """a_*: bf16 [NI, AH, AW, Cin]; w_*: bf16 [T, Cout, Cin]; taps: list of (dy, dx, img_off, wtap)."""
    p = _conv_desc(a_hi, a_lo, w_hi, w_lo, N, MH, MW, nprod)
    p.a_img_mul = a_img_mul
    p.ntaps = len(taps)
    for i, (dy, dx, io, wt) in enumerate(taps):
        p.taps[i] = _lib.ConvTap(dy, dx, io, wt)
    p.mode = mode
    p.dcoef, p.bias, p.noise, p.noise_nstride = ptr(dcoef), ptr(bias), ptr(noise), noise_nstride
    p.gain, p.slope, p.clamp = gain, slope, clamp
    for i, o in enumerate(outs):
        p.out[i] = o
    p.out_f32 = ptr(out_f32)
    p.f32_cstride, p.f32_coff, p.f32_nchw, p.f32_accumulate = f32_cstride, f32_coff, int(f32_nchw), int(f32_accumulate)
    p.oy_mul, p.oy_off, p.ox_mul, p.ox_off = oy_mul, oy_off, ox_mul, ox_off
    p.OH = OH if OH is not None else MH * oy_mul
    p.OW = OW if OW is not None else MW * ox_mul
    if rgb is not None:                                  # dict(out, weight [c,Cout], style [N,Cout], bias [c], clamp, nchw, accumulate)
        p.rgb = _lib.FusedRgb(ptr(rgb['out']), ptr(rgb['weight']), ptr(rgb['style']), ptr(rgb['bias']), float(rgb.get('clamp', -1.0)),
                              rgb['weight'].shape[0], int(rgb.get('nchw', False)), int(rgb.get('accumulate', False)))
    p.splits, p.split_stride = splits, split_stride
    _run('n3d_conv_gemm', C.byref(p), stream_ptr())


def conv_transposed_gemm(a_hi, a_lo, w_hi, w_lo, N, H, W, raw, nprod=3):
    """Stride-2 transposed 3x3 conv of a [N,H,W,Cin] split activation -> raw fp32 [N,2H+1,2W+1,Cout] (one launch, 4 parity classes)."""
    p = _conv_desc(a_hi, a_lo, w_hi, w_lo, N, H, W, nprod)
    p.gain, p.slope, p.clamp = 1.0, 1.0, -1.0
    p.out_f32, p.f32_cstride = ptr(raw), raw.shape[-1]
    _run('n3d_conv_transposed_gemm', C.byref(p), stream_ptr())


def wgrad_operand(x, s, pt, pl, PH, PW, ld, hi, lo, shift=0):
    """x fp32 [N, C, H, W] (any strides) -> channel-major split operand hi / lo bf16 [C, ld] of conv_wgrad: column
    ((par * N + n) * PH + py) * PW + px - shift holds x[n, c, s*(py - pt) + par // s, s*(px - pl) + par % s] (0 elsewhere)."""
    N, Cc, H, W = x.shape
    _run('n3d_wgrad_operand', ptr(x), (_lib.I64 * 4)(*x.stride()), N, Cc, H, W, s, pt, pl, PH, PW, shift, ld, ptr(hi), ptr(lo), stream_ptr())


def wgrad_splits(G, T, M, N, K):
    """K slices of a conv_wgrad launch: about two waves of CTAs over the device's SMs, at least 8 K steps (of 64 positions) per slice.
    A function of the shapes and the SM count only, so the same call always sums in the same order."""
    bn = 32 if N <= 32 else 64 if N <= 64 else 128
    tiles = -(-M // 128) * -(-N // bn) * T * G
    ksteps = K // 64
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return max(1, min(max(ksteps // 8, 1), -(-2 * sms // tiles)))


def conv_wgrad(a_hi, a_lo, b_hi, b_lo, G, M, N, K, a_off, b_off, dw, splits=1, partial=None, a_cols=None, b_cols=None, a_row=None, b_row=None):
    """dw fp32 [G, T, M, N] = sum_{k < K} A[a_row[t] + g*M + m, k + a_off[t]] * B[b_row[t] + g*N + n, k + b_off[t]] (a_*: bf16
    [rows, lda], b_*: bf16 [rows, ldb], columns outside [0, a_cols) / [0, b_cols) (default: the row length) read as 0; column offsets
    are multiples of 8, row offsets default to 0).  splits > 1 needs partial fp32 [splits, G, T, M, N]."""
    p = _lib.ConvWgrad()
    p.a_hi, p.a_lo, p.a_rows, p.lda = ptr(a_hi), ptr(a_lo), a_hi.shape[0], a_hi.shape[1]
    p.a_cols = a_hi.shape[1] if a_cols is None else a_cols
    p.b_hi, p.b_lo, p.b_rows, p.ldb = ptr(b_hi), ptr(b_lo), b_hi.shape[0], b_hi.shape[1]
    p.b_cols = b_hi.shape[1] if b_cols is None else b_cols
    p.G, p.M, p.N, p.T, p.K = G, M, N, len(a_off), K
    for t, (ao, bo) in enumerate(zip(a_off, b_off)):
        p.a_off[t], p.b_off[t] = ao, bo
        p.a_row[t] = a_row[t] if a_row is not None else 0
        p.b_row[t] = b_row[t] if b_row is not None else 0
    p.splits, p.partial, p.dw = splits, ptr(partial), ptr(dw)
    _run('n3d_conv_wgrad', C.byref(p), stream_ptr(), kernels=1 if splits == 1 else 2)


def modulate_split(x, style, hi, lo, cstride=None, coff=0):
    """x fp32 NHWC [N,H,W,C]; style [N,C] or None -> hi/lo bf16 (written at channel offset `coff`, stride `cstride`)."""
    N, H, W, Cc = x.shape
    _run('n3d_modulate_split', ptr(x), H * W, N, Cc, ptr(style), ptr(hi), ptr(lo), cstride or Cc, coff, stream_ptr())


def modulate_f16(x, style, out, cstride=None, coff=0):
    """x fp32 NHWC [N,H,W,C]; style [N,C] or None -> out fp16 = x * style (channel offset `coff`, stride `cstride`)."""
    N, H, W, Cc = x.shape
    _run('n3d_modulate_f16', ptr(x), H * W, N, Cc, ptr(style), ptr(out), cstride or Cc, coff, stream_ptr())


def fir_up_epilogue(raw, C_, dcoef, bias, noise, gain, slope, clamp, outs=(), out_f32=None, f32_cstride=0, f32_coff=0, noise_nstride=0):
    N, RH, RW, _ = raw.shape
    arr = (_lib.SplitOut * 2)()
    for i, o in enumerate(outs):
        arr[i] = o
    _run('n3d_fir_up_epilogue', ptr(raw), N, RH - 1, RW - 1, C_, ptr(dcoef), ptr(bias), ptr(noise), noise_nstride, gain, slope, clamp, arr,
                                ptr(out_f32), f32_cstride, f32_coff, stream_ptr())


def splitk_epilogue(part, dcoef, bias, noise, gain, slope, clamp, outs=(), out_f32=None, f32_cstride=0, f32_coff=0, noise_nstride=0):
    """part: fp32 [S, N, H, W, C] raw partial sums of a split-K conv_gemm (mode 1) -> summed, then the mode-0 epilogue."""
    S, N, H, W, Cc = part.shape
    arr = (_lib.SplitOut * 2)()
    for i, o in enumerate(outs):
        arr[i] = o
    _run('n3d_splitk_epilogue', ptr(part), S, N * H * W * Cc, N, H, W, Cc, ptr(dcoef), ptr(bias), ptr(noise), noise_nstride, gain, slope, clamp, arr,
                                ptr(out_f32), f32_cstride, f32_coff, stream_ptr())


def fir_down_split(x, hi, lo):
    N, H, W, Cc = x.shape
    _run('n3d_fir_down_split', ptr(x), N, H, W, Cc, ptr(hi), ptr(lo), stream_ptr())


def upsample2d_nhwc(x, y, y_nchw=False):
    N, H, W, Cc = x.shape
    _run('n3d_upsample2d_nhwc', ptr(x), N, H, W, Cc, ptr(y), int(y_nchw), stream_ptr())


def downsample2d_nhwc(x, y):
    N, H, W, Cc = x.shape
    _run('n3d_downsample2d_nhwc', ptr(x), N, H, W, Cc, ptr(y), stream_ptr())


def styles(ws, affine_w, affine_b, row_widx, row_scale, row_ooff, row_cin, out):
    """out: flat fp32; layer blocks are dense [N, Cin] at row_ooff (see include/next3d_b200.h)."""
    N, num_ws, wdim = ws.shape
    rows = affine_w.shape[0]
    _run('n3d_styles', ptr(ws), N, num_ws, wdim, ptr(affine_w), ptr(affine_b), ptr(row_widx), ptr(row_scale), ptr(row_ooff),
                       ptr(row_cin), ptr(out), rows, stream_ptr())


def demod(styles_flat, wsq, row_woff, row_cin, row_soff, row_ooff, row_cout, out, N):
    rows = row_cin.shape[0]
    _run('n3d_demod', ptr(styles_flat), ptr(wsq), ptr(row_woff), ptr(row_cin), ptr(row_soff), ptr(row_ooff), ptr(row_cout),
                      ptr(out), rows, N, stream_ptr())


def transform_points(pts, rot, zoff, ndc_flip, out):
    N, Pn, _ = pts.shape
    _run('n3d_transform_points', ptr(pts), N, Pn, ptr(rot), rot.shape[0], zoff, int(ndc_flip), ptr(out), stream_ptr())


def rasterize(verts, faces, H, W, p2f, bary, workspace=None):
    NM, V, _ = verts.shape
    if workspace is None:
        workspace = torch.empty(NM * faces.shape[0] * 16, dtype=torch.float32, device=verts.device)
    _run('n3d_rasterize', ptr(verts), ptr(faces), NM, V, faces.shape[0], H, W, ptr(p2f), ptr(bary), ptr(workspace), stream_ptr(), kernels=2)


def uv_sample(p2f, bary, face_uv, texture, eye_mask, tex_planes, alpha, views=1):
    """views: images per texture -- N = texture.shape[0] * views images, image n reads texture n // views."""
    B, TH, TW, Cc = texture.shape
    _, H, W = p2f.shape
    MH, MW = eye_mask.shape[-2:]
    _run('n3d_uv_sample_views', ptr(p2f), ptr(bary), ptr(face_uv), ptr(texture), ptr(eye_mask), B * views, views, H, W, TH, TW, Cc, MH, MW,
                                ptr(tex_planes), ptr(alpha), stream_ptr())


def fill_mouth(alpha, binarize=(0, 0)):
    """alpha [..., H, W] in place; the images [binarize[0], binarize[1]) of the flattened leading dims end as (alpha != 0)."""
    NI = alpha.numel() // (alpha.shape[-1] * alpha.shape[-2])
    if binarize[0] == binarize[1]:
        _run('n3d_fill_mouth', ptr(alpha), NI, alpha.shape[-2], alpha.shape[-1], stream_ptr())
    else:
        _run('n3d_fill_mouth_binarize', ptr(alpha), NI, alpha.shape[-2], alpha.shape[-1], binarize[0], binarize[1], stream_ptr())


def mouth_box(lm2d, boxes):
    _run('n3d_mouth_box', ptr(lm2d), lm2d.shape[0], ptr(boxes), stream_ptr())


def resize_aa(src, dst=None, DH=None, DW=None, src_box=None, dst_box=None, style=None, hi=None, lo=None):
    N, SH, SW, Cc = src.shape
    if dst is not None:
        DH, DW = dst.shape[1:3]
    _run('n3d_resize_aa', ptr(src), N, SH, SW, Cc, ptr(src_box), ptr(dst), DH, DW, ptr(dst_box), ptr(style), ptr(hi), ptr(lo),
                          stream_ptr())


def resize_aa_f16(src, out, src_box=None, dst_box=None, style=None):
    """resize_aa into the fp16 NHWC tensor out [N, DH, DW, C] only: out = fp16(resize(src) * style)."""
    N, SH, SW, Cc = src.shape
    DH, DW = out.shape[1:3]
    _run('n3d_resize_aa_f16', ptr(src), N, SH, SW, Cc, ptr(src_box), DH, DW, ptr(dst_box), ptr(style), ptr(out), stream_ptr())


def blend_planes(front, tex_planes, alpha, static, planes, views=1):
    """views: images per static plane set -- image n of front's N reads static n // views."""
    N, H, W, _ = front.shape
    _run('n3d_blend_planes_views', ptr(front), ptr(tex_planes), ptr(alpha), ptr(static), N, views, H, W, ptr(planes), stream_ptr())


def _render_desc(planes, cam2world, intrinsics, res, opts, seed, views=1):
    """Render descriptor with the workload (planes, cameras, resolution, sampling options, seed) filled in: views images per plane set,
    so planes.shape[0] * views images."""
    p = _lib.Render()
    B, _, PH, PW, _ = planes.shape
    p.planes, p.N, p.PH, p.PW, p.views = ptr(planes), B * max(views, 1), PH, PW, views
    p.cam2world, p.intrinsics, p.res = ptr(cam2world), ptr(intrinsics), res
    p.depth_coarse, p.depth_fine = opts['depth_resolution'], opts['depth_resolution_importance']
    p.ray_start, p.ray_end, p.box_warp = float(opts['ray_start']), float(opts['ray_end']), float(opts['box_warp'])
    p.ray_span = float(opts['ray_end']) - float(opts['ray_start'])        # the jitter spacing's numerator, in double as the reference has it
    p.seed = seed_bits(seed)
    return p


SEED_MASK = (1 << 64) - 1


def seed_bits(seed):
    """The sampler seed as the renderer uses it: its 64-bit pattern, so any integer is accepted and seeds equal modulo 2^64 (-1 and
    2^64 - 1, say) draw the same uniforms."""
    return int(seed) & SEED_MASK


def check_render_options(opts):
    """Raise for the rendering options the fused renderer lacks.  Every render call runs this first, the graph-replayed ones too (a
    replay runs no Python of the call it captured)."""
    unsupported = [k for k, bad in (('disparity_space_sampling', bool(opts.get('disparity_space_sampling', False))),
                                    ('density_noise', float(opts.get('density_noise', 0) or 0) > 0),
                                    ('clamp_mode', opts.get('clamp_mode', 'softplus') != 'softplus'),
                                    ('ray_start/ray_end', isinstance(opts.get('ray_start'), str) or isinstance(opts.get('ray_end'), str))) if bad]
    if unsupported:     # renderer.py:98-107 (auto near/far), :153 (density noise), :186-196 (disparity sampling), ray_marcher.py:41-44
        raise RuntimeError(f'libnext3d_b200 n3d_render_rays failed (code -2, unsupported): rendering option(s) {unsupported} are not '
                           f'implemented by the fused renderer (supported: linear stratified sampling, fixed ray_start / ray_end, softplus)')


def _render_full_desc(planes, cam2world, intrinsics, res, opts, dec, rgb, depth, wsum, depth_minmax, u_coarse, u_fine, seed, seed_ptr, views=1,
                      depth_range_per_image=0):
    """Render descriptor of n3d_render_rays / n3d_render_rays_normals, after rejecting the rendering options the renderer lacks."""
    check_render_options(opts)
    p = _render_desc(planes, cam2world, intrinsics, res, opts, seed, views)
    p.u_coarse, p.u_fine, p.seed_ptr = ptr(u_coarse), ptr(u_fine), ptr(seed_ptr)
    p.w0, p.b0, p.w1, p.b1 = (ptr(t) for t in dec)
    p.rgb, p.depth, p.wsum, p.depth_minmax = ptr(rgb), ptr(depth), ptr(wsum), ptr(depth_minmax)
    p.white_back = int(bool(opts.get('white_back', False)))
    p.depth_range_per_image = depth_range_per_image
    return p


def render_rays(planes, cam2world, intrinsics, res, opts, dec, rgb, depth, wsum, depth_minmax, u_coarse=None, u_fine=None, seed=0,
                seed_ptr=None, views=1, depth_range_per_image=0):
    """planes [B,3,PH,PW,32] channels-last; dec = (w0 [64,32], b0 [64], w1 [33,64], b1 [33]) with gains folded in.
    opts['depth_resolution'] (4 .. 192) and opts['depth_resolution_importance'] (0 = coarse only .. 192) are samples per pass; a
    count above 192 raises (code -2, unsupported).  views: camera views per plane set -- N = B * views images, image n reads plane
    set n // views; cameras, uniforms and outputs are per image.  depth_range_per_image=1: depth_minmax is [N, 2] (each pair
    initialised to (+inf, -inf)) and pair n covers image n's samples only; 0: depth_minmax [2] covers the launch."""
    p = _render_full_desc(planes, cam2world, intrinsics, res, opts, dec, rgb, depth, wsum, depth_minmax, u_coarse, u_fine, seed, seed_ptr,
                          views, depth_range_per_image)
    _run('n3d_render_rays', C.byref(p), stream_ptr())


def normals_workspace_floats(N, res, opts):
    """Floats of the n3d_render_rays_normals workspace: N * M * (2D - 1), D = samples per ray after the merge."""
    Dc, Df = opts['depth_resolution'], opts['depth_resolution_importance']
    return N * res * res * (2 * (Dc + Df if Df > 0 else Dc) - 1)


def render_rays_normals(planes, cam2world, intrinsics, res, opts, dec, rgb, depth, wsum, depth_minmax, normal, workspace=None, u_coarse=None,
                        u_fine=None, seed=0, seed_ptr=None, views=1, depth_range_per_image=0):
    """render_rays (same outputs, bit for bit) plus normal [N, M, 3]: unit world-space normals -grad sigma composited with the final
    weights (rendering option return_normal).  workspace: fp32 device buffer of normals_workspace_floats() floats, or None to
    allocate one here.  Same sample-count limits, `views` and `depth_range_per_image` as render_rays (N = planes.shape[0] * views
    images)."""
    p = _render_full_desc(planes, cam2world, intrinsics, res, opts, dec, rgb, depth, wsum, depth_minmax, u_coarse, u_fine, seed, seed_ptr,
                          views, depth_range_per_image)
    n_ws = normals_workspace_floats(p.N, res, opts)
    if workspace is None:
        workspace = torch.empty(n_ws, dtype=torch.float32, device=planes.device)
    elif workspace.numel() < n_ws or workspace.dtype != torch.float32:
        raise RuntimeError(f'render_rays_normals: workspace needs {n_ws} float32 elements, got {workspace.numel()} {workspace.dtype}')
    if normal.numel() != p.N * res * res * 3 or normal.dtype != torch.float32:
        raise RuntimeError(f'render_rays_normals: normal must be float32 [N, M, 3], got {tuple(normal.shape)} {normal.dtype}')
    _run('n3d_render_rays_normals', C.byref(p), ptr(normal), ptr(workspace), stream_ptr(), kernels=2)


def render_normals_pass(planes, cam2world, intrinsics, res, opts, dec, normal, workspace):
    """Diagnostics (n3d_render_normals_pass): the normal pass alone over the samples an earlier render_rays_normals call with the same
    workload left in `workspace`."""
    p = _render_desc(planes, cam2world, intrinsics, res, opts, 0)
    p.w0, p.b0, p.w1, p.b1 = (ptr(t) for t in dec)
    p.rgb = p.depth = p.wsum = ptr(normal)         # not written; the argument checks are n3d_render_rays'
    _run('n3d_render_normals_pass', C.byref(p), ptr(workspace), ptr(normal), stream_ptr())


def depth_clamp(depth, depth_minmax):
    _run('n3d_depth_clamp', ptr(depth), depth.numel(), ptr(depth_minmax), stream_ptr())


def depth_clamp_images(depth, depth_minmax):
    """Clamp image n of depth [N, ...] to its own range depth_minmax[n] of depth_minmax [N, 2] (render_rays with
    depth_range_per_image=1)."""
    N = depth.shape[0]
    if depth_minmax.numel() != 2 * N:
        raise RuntimeError(f'depth_clamp_images: depth_minmax must be [{N}, 2], got {tuple(depth_minmax.shape)}')
    _run('n3d_depth_clamp_images', ptr(depth), N, depth.numel() // max(N, 1), ptr(depth_minmax), stream_ptr())


POINT_FEATURES = 32            # channels n3d_sample_points writes per point (the decoder's output after sigma)


def sample_points(planes, coords, box_warp, dec, sigma, rgb=None):
    N, _, PH, PW, _ = planes.shape
    Pn = coords.shape[1]
    _run('n3d_sample_points', ptr(planes), N, PH, PW, ptr(coords), Pn, float(box_warp), *(ptr(t) for t in dec), ptr(sigma), ptr(rgb),
                              stream_ptr())


def sample_grid(planes, grid_n, cube_length, box_warp, dec, sigma_grid, head=0, count=None, pad=0, pad_value=-1000.0):
    """sigma of the create_samples voxel grid (in-kernel coordinates), written flipped + trimmed into sigma_grid [grid_n]^3."""
    _, PH, PW, _ = planes.shape[-4:]
    count = grid_n ** 3 - head if count is None else count
    _run('n3d_sample_grid', ptr(planes), PH, PW, grid_n, float(cube_length), float(box_warp), head, count, pad, float(pad_value),
                            *(ptr(t) for t in dec), ptr(sigma_grid), stream_ptr())


def mapping_cutoff(truncation_cutoff, num_ws):
    """The layers the reference truncates, ws[:, :truncation_cutoff] (networks_stylegan2.py:267; None: all of them), as n3d_mapping's
    count of leading layers (< 0: all): a negative cutoff leaves its last -cutoff layers untruncated, as the slice does."""
    if truncation_cutoff is None:
        return -1
    c = int(truncation_cutoff)
    return max(num_ws + c, 0) if c < 0 else c


def mapping(z, c, c_scale, m, truncation_psi=1.0, truncation_cutoff=None, num_ws=28, out=None):
    """MappingNetwork + truncation in one launch.  m: dict with embed_w/embed_b/fc0_w/fc0_b/fc1_w/fc1_b/w_avg fp32 device tensors.
    out: the [N, num_ws, 512] result, allocated when None."""
    N = z.shape[0]
    ws = torch.empty(N, num_ws, 512, device=z.device, dtype=torch.float32) if out is None else out
    _run('n3d_mapping', ptr(z), ptr(c), N, float(c_scale), ptr(m['embed_w']), ptr(m['embed_b']), ptr(m['fc0_w']), ptr(m['fc0_b']),
                        ptr(m['fc1_w']), ptr(m['fc1_b']), ptr(m['w_avg']), float(truncation_psi),
                        mapping_cutoff(truncation_cutoff, num_ws), num_ws, ptr(ws), stream_ptr())
    return ws


def interp_rows(B, Y, out=None):
    """out[f] = sum_k B[f,k] * Y[k] for fp32 device tensors B [F,K], Y [K, ...] -> [F, ...] (allocated when out is None)."""
    F_, K_ = B.shape
    D = Y[0].numel()
    if out is None:
        out = torch.empty((F_,) + tuple(Y.shape[1:]), device=Y.device, dtype=torch.float32)
    _run('n3d_interp_rows', ptr(B), ptr(Y), F_, K_, D, ptr(out), stream_ptr())
    return out


def render_floor(planes, cam2world, intrinsics, res, opts, kind, seed=0):
    """Diagnostics (n3d_render_floor): launch the gather-only (kind 0) or activations-only (kind 1) micro-kernel on the renderer's workload."""
    p = _render_desc(planes, cam2world, intrinsics, res, opts, seed)
    _run('n3d_render_floor', C.byref(p), int(kind), None, stream_ptr())
