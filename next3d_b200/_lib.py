"""ctypes binding of libnext3d_b200.so (the C ABI declared in include/next3d_b200.h).

The shared library is mandatory: there is no CPU / PyTorch fallback anywhere in this package.  Importing this module
without the built library raises immediately (run `python -c "import __graft_entry__ as g; g.build()"` or
`make -C next3d_b200/csrc`).
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('N3D_LIB_PATH') or os.path.join(_HERE, 'libnext3d_b200.so')      # N3D_LIB_PATH: A/B builds of the same library (tools only)

if not os.path.exists(LIB_PATH):
    raise ImportError(f'{LIB_PATH} is missing: build it with `make -C {os.path.join(_HERE, "csrc")}` '
                      '(next3d_b200 has no fallback path)')

lib = C.CDLL(LIB_PATH)

P = C.c_void_p
I32, I64, F32 = C.c_int32, C.c_int64, C.c_float


class ConvTap(C.Structure):
    _fields_ = [('dy', C.c_int8), ('dx', C.c_int8), ('img_off', C.c_int16), ('wtap', C.c_int32)]


class SplitOut(C.Structure):
    _fields_ = [('hi', P), ('lo', P), ('style', P), ('cstride', I32), ('coff', I32), ('f16', I32)]


class FusedRgb(C.Structure):
    _fields_ = [('out', P), ('weight', P), ('style', P), ('bias', P), ('clamp', F32), ('channels', I32), ('nchw', I32), ('accumulate', I32)]


class ConvGemm(C.Structure):
    _fields_ = [
        ('a_hi', P), ('a_lo', P), ('NI', I32), ('AH', I32), ('AW', I32), ('Cin', I32),
        ('w_hi', P), ('w_lo', P), ('T', I32), ('Cout', I32),
        ('N', I32), ('MH', I32), ('MW', I32), ('a_img_mul', I32),
        ('ntaps', I32), ('taps', ConvTap * 9),
        ('nprod', I32), ('mode', I32),
        ('dcoef', P), ('bias', P), ('noise', P), ('noise_nstride', I64),
        ('gain', F32), ('slope', F32), ('clamp', F32),
        ('out', SplitOut * 2),
        ('out_f32', P), ('f32_cstride', I32), ('f32_coff', I32), ('f32_nchw', I32), ('f32_accumulate', I32),
        ('oy_mul', I32), ('oy_off', I32), ('ox_mul', I32), ('ox_off', I32), ('OH', I32), ('OW', I32),
        ('rgb', FusedRgb),
        ('splits', I32), ('split_stride', I64),
        ('f16', I32),
    ]


class ConvWgrad(C.Structure):
    _fields_ = [
        ('a_hi', P), ('a_lo', P), ('a_rows', I32), ('a_cols', I64), ('lda', I64),
        ('b_hi', P), ('b_lo', P), ('b_rows', I32), ('b_cols', I64), ('ldb', I64),
        ('G', I32), ('M', I32), ('N', I32), ('T', I32), ('K', I64),
        ('a_off', I64 * 9), ('b_off', I64 * 9), ('a_row', I32 * 9), ('b_row', I32 * 9),
        ('splits', I32), ('partial', P), ('dw', P),
    ]


class Render(C.Structure):
    _fields_ = [
        ('planes', P), ('N', I32), ('PH', I32), ('PW', I32),
        ('cam2world', P), ('intrinsics', P), ('res', I32), ('depth_coarse', I32), ('depth_fine', I32),
        ('ray_start', F32), ('ray_end', F32), ('box_warp', F32),
        ('u_coarse', P), ('u_fine', P), ('seed', C.c_uint64), ('seed_ptr', P),
        ('w0', P), ('b0', P), ('w1', P), ('b1', P),
        ('rgb', P), ('depth', P), ('wsum', P), ('depth_minmax', P), ('white_back', I32), ('views', I32), ('depth_range_per_image', I32),
        ('ray_span', C.c_double),
    ]


_SIGNATURES = {
    'n3d_version': ([], C.c_int),
    'n3d_last_error': ([], C.c_char_p),
    'n3d_bias_act': ([P, P, P, C.c_int, I64, C.c_int, C.c_int, C.c_int, F32, F32, F32, P], C.c_int),
    'n3d_bias_act_grad': ([P, P, P, P, P, P, C.c_int, I64, C.c_int, C.c_int, C.c_int, C.c_int, F32, F32, F32, P], C.c_int),
    'n3d_upfirdn2d': ([P, P, P, C.c_int] + [C.c_int] * 4 + [C.POINTER(I64), C.POINTER(I64)] + [C.c_int] * 10 + [C.c_int, F32, C.c_int, C.c_int, P], C.c_int),
    'n3d_filtered_lrelu': ([P, P, P, P, P, P, C.c_int] + [C.c_int] * 14 + [F32, F32, F32, C.c_int, C.c_int, C.c_int, P], C.c_int),
    'n3d_styles': ([P, C.c_int, C.c_int, C.c_int, P, P, P, P, P, P, P, C.c_int, P], C.c_int),
    'n3d_demod': ([P, P, P, P, P, P, P, P, C.c_int, C.c_int, P], C.c_int),
    'n3d_conv_gemm': ([C.POINTER(ConvGemm), P], C.c_int),
    'n3d_conv_transposed_gemm': ([C.POINTER(ConvGemm), P], C.c_int),
    'n3d_conv_wgrad': ([C.POINTER(ConvWgrad), P], C.c_int),
    'n3d_wgrad_operand': ([P, C.POINTER(I64)] + [C.c_int] * 10 + [I64, P, P, P], C.c_int),
    'n3d_modulate_split': ([P, I64, C.c_int, C.c_int, P, P, P, C.c_int, C.c_int, P], C.c_int),
    'n3d_modulate_f16': ([P, I64, C.c_int, C.c_int, P, P, C.c_int, C.c_int, P], C.c_int),
    'n3d_fir_up_epilogue': ([P, C.c_int, C.c_int, C.c_int, C.c_int, P, P, P, I64, F32, F32, F32, C.POINTER(SplitOut), P, C.c_int, C.c_int, P], C.c_int),
    'n3d_parse_obj_vertices': ([C.c_char_p, I64, P, I64, C.POINTER(I64)], C.c_int),
    'n3d_parse_float_table': ([C.c_char_p, I64, P, I64, C.POINTER(I64), C.POINTER(I64)], C.c_int),
    'n3d_splitk_epilogue': ([P, C.c_int, I64, C.c_int, C.c_int, C.c_int, C.c_int, P, P, P, I64, F32, F32, F32, C.POINTER(SplitOut), P, C.c_int, C.c_int, P], C.c_int),
    'n3d_fir_down_split': ([P, C.c_int, C.c_int, C.c_int, C.c_int, P, P, P], C.c_int),
    'n3d_upsample2d_nhwc': ([P, C.c_int, C.c_int, C.c_int, C.c_int, P, C.c_int, P], C.c_int),
    'n3d_downsample2d_nhwc': ([P, C.c_int, C.c_int, C.c_int, C.c_int, P, P], C.c_int),
    'n3d_transform_points': ([P, C.c_int, C.c_int, P, C.c_int, F32, C.c_int, P, P], C.c_int),
    'n3d_rasterize': ([P, P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, P, P, P, P], C.c_int),
    'n3d_uv_sample': ([P, P, P, P, P] + [C.c_int] * 8 + [P, P, P], C.c_int),
    'n3d_uv_sample_views': ([P, P, P, P, P] + [C.c_int] * 9 + [P, P, P], C.c_int),
    'n3d_fill_mouth': ([P, C.c_int, C.c_int, C.c_int, P], C.c_int),
    'n3d_fill_mouth_binarize': ([P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, P], C.c_int),
    'n3d_mouth_box': ([P, C.c_int, P, P], C.c_int),
    'n3d_resize_aa': ([P, C.c_int, C.c_int, C.c_int, C.c_int, P, P, C.c_int, C.c_int, P, P, P, P, P], C.c_int),
    'n3d_resize_aa_f16': ([P, C.c_int, C.c_int, C.c_int, C.c_int, P, C.c_int, C.c_int, P, P, P, P], C.c_int),
    'n3d_blend_planes': ([P, P, P, P, C.c_int, C.c_int, C.c_int, P, P], C.c_int),
    'n3d_blend_planes_views': ([P, P, P, P, C.c_int, C.c_int, C.c_int, C.c_int, P, P], C.c_int),
    'n3d_render_rays': ([C.POINTER(Render), P], C.c_int),
    'n3d_render_rays_normals': ([C.POINTER(Render), P, P, P], C.c_int),
    'n3d_render_normals_pass': ([C.POINTER(Render), P, P, P], C.c_int),
    'n3d_depth_clamp': ([P, I64, P, P], C.c_int),
    'n3d_depth_clamp_images': ([P, C.c_int, I64, P, P], C.c_int),
    'n3d_sample_points': ([P, C.c_int, C.c_int, C.c_int, P, I64, F32, P, P, P, P, P, P, P], C.c_int),
    'n3d_bake_world_points': ([P, I64, C.c_int, F32, P, P], C.c_int),
    'n3d_mesh_zbuffer': ([P, I64, P, I64, P, P, C.c_int, C.c_int, C.c_int, F32, P, P], C.c_int),
    'n3d_bake_vertex_colors': ([P, P, I64, P, C.c_int, P, P, C.c_int, P, C.c_int, C.c_int, P, F32, F32, P, C.c_int, P, P, P, P], C.c_int),
    'n3d_render_floor': ([P, C.c_int, P, P], C.c_int),
    'n3d_mapping': ([P, P, C.c_int, F32, P, P, P, P, P, P, P, F32, C.c_int, C.c_int, P, P], C.c_int),
    'n3d_interp_rows': ([P, P, C.c_int, C.c_int, I64, P, P], C.c_int),
    'n3d_h264_buffer_sizes': ([C.c_int, C.c_int, C.POINTER(I64), C.POINTER(I64), C.POINTER(I64), C.POINTER(I64)], C.c_int),
    'n3d_h264_encode': ([P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, P, P, P, P, P, P, P, P], C.c_int),
    'n3d_h264_rc_init': ([P, C.c_int, C.c_int, I64, C.c_int, C.c_int, C.c_int, C.c_int, P], C.c_int),
    'n3d_h264_encode_rc': ([P, C.c_int, C.c_int, P, C.c_int, C.c_int, C.c_int, P, P, P, P, P, P, P, P], C.c_int),
    'n3d_png_buffer_sizes': ([C.c_int, C.c_int, C.c_int, C.POINTER(I64), C.POINTER(I64)], C.c_int),
    'n3d_png_encode': ([P, C.c_int, C.c_int, C.c_int, P, P, P, P], C.c_int),
    'n3d_isosurface_workspace_bytes': ([C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)], C.c_int),
    'n3d_isosurface_count': ([P, C.c_int, C.c_int, C.c_int, F32, P, P, P], C.c_int),
    'n3d_isosurface_emit': ([P, C.c_int, C.c_int, C.c_int, F32, P, P, P, P], C.c_int),
    'n3d_sample_grid': ([P, C.c_int, C.c_int, C.c_int, F32, F32, I64, I64, C.c_int, F32, P, P, P, P, P, P], C.c_int),
}

EXPORTS = sorted(_SIGNATURES)
H264_RC_STATE_BYTES = 128             # N3D_H264_RC_STATE_BYTES

for _name, (_args, _res) in _SIGNATURES.items():
    _fn = getattr(lib, _name)          # AttributeError here = the library does not export what the header declares
    _fn.argtypes = _args
    _fn.restype = _res


def check(rc, what=''):
    if rc != 0:
        raise RuntimeError(f'libnext3d_b200 {what} failed (code {rc}): {lib.n3d_last_error().decode()}')


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


def stream_ptr(device=None):
    return torch.cuda.current_stream(device).cuda_stream


def require_cuda(t, name='tensor'):
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise RuntimeError(f'next3d_b200: {name} must be a CUDA tensor (there is no CPU path in this package)')
