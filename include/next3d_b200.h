/* libnext3d_b200.so -- C ABI of the Hopper-native (sm_90a) Next3D generator hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b).  The reference reaches its native code through three pybind11
 * plugins JIT-built by torch_utils/custom_ops.py:61 (`get_plugin`):
 *     bias_act_plugin.bias_act              torch_utils/ops/bias_act.cpp:36,100
 *     upfirdn2d_plugin.upfirdn2d            torch_utils/ops/upfirdn2d.cpp:20,108
 *     filtered_lrelu_plugin.filtered_lrelu  torch_utils/ops/filtered_lrelu.cpp:20,300
 * and runs everything else (modulated conv, rasterizer, grid_sample, volume renderer) through ATen /
 * cuDNN / pytorch3d / OpenCV calls.  This library replaces all of it with plain-C entry points:
 * raw device pointers + sizes in, int status out, no torch / C++ types, caller-owned buffers, explicit stream,
 * no allocation, no host sync and no global mutable device state inside (CUDA-graph capturable).
 *
 * Conventions
 *   - return value: 0 = ok, <0 = error (N3D_ERR_*); n3d_last_error() returns a thread-local message.
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream).
 *   - "NHWC" = channels-last [N,H,W,C]; "split bf16" = two bf16 tensors (hi, lo) with hi+lo ~= the fp32 value
 *     (operands of the 3-product bf16 tensor-core scheme, see DESIGN.md).  "fp16 single" = one fp16 tensor: the operands of
 *     the opt-in fp16 super-resolution head (one product per k-step), which the reference runs in fp16 on CUDA
 *     (superresolution.py:268-277, networks_stylegan2.py:547-549 with sr_num_fp16_res > 0).
 */
#ifndef NEXT3D_B200_H
#define NEXT3D_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define N3D_OK 0
#define N3D_ERR_INVALID_ARG (-1)
#define N3D_ERR_UNSUPPORTED (-2)
#define N3D_ERR_CUDA (-3)

#define N3D_DTYPE_F32 0
#define N3D_DTYPE_F16 1

const char* n3d_last_error(void);
int n3d_version(void);

/* ------------------------------------------------------------------------------------------------------------
 * Op-level API: the native half of torch_utils.ops (NCHW or channels_last tensors described by element strides).
 * ---------------------------------------------------------------------------------------------------------- */

/* y = clamp(act(x + b[(i / step_b) % size_b]) * gain, +-clamp)   -- replaces bias_act_plugin.bias_act
 * (bias_act.cpp:36-94, kernel bias_act.cu:28-151; forward, grad == 0; the grad modes are n3d_bias_act_grad).  act: 1 linear, 2 relu, 3 lrelu,
 * 4 tanh, 5 sigmoid, 6 elu, 7 selu, 8 softplus, 9 swish (the reference's cuda_idx, bias_act.py:23-33).
 * x dense (any memory format), b contiguous or NULL, clamp < 0 disables clamping.  x and y may start anywhere (a view into a larger
 * storage): 4-element vector accesses are used only when both are aligned for them (16 bytes fp32, 8 bytes fp16). */
int n3d_bias_act(const void* x, const void* b, void* y, int dtype, int64_t numel, int size_b, int step_b,
                 int act, float alpha, float gain, float clamp, void* stream);

/* Gradients of n3d_bias_act: the plugin's grad modes 1 and 2 (bias_act.cu:58-146, called from BiasActCudaGrad, bias_act.py:177-205).
 *   grad 1: dx = dy * act'(xref + b) * gain, with act' taken from yref / gain (act 2-8) or from xref + b (act 9, swish);
 *   grad 2: dx = dy * act''(xref + b) * gain * dyref (act 4-9 only: the activations with a second derivative).
 * Elements whose saved output lies on or outside +-clamp (clamp >= 0) get 0; swish recomputes that output from xref + b.
 * dy, xref, yref, dyref and dx share x's dense layout; b is applied to xref only.  xref is required for act 9, yref for act 2-8
 * (a NULL yref counts as 0, as in the plugin, so `linear` with a clamp passes every element), dyref for grad 2.  numel 0 launches
 * nothing and accepts NULL pointers (an empty tensor's data pointer). */
int n3d_bias_act_grad(const void* dy, const void* b, const void* xref, const void* yref, const void* dyref, void* dx, int dtype,
                      int64_t numel, int size_b, int step_b, int grad, int act, float alpha, float gain, float clamp, void* stream);

/* Zero-insert upsample -> pad/crop -> 2-D FIR -> decimate, per (n,c) plane  -- replaces upfirdn2d_plugin.upfirdn2d
 * (upfirdn2d.cpp:20-102, kernels upfirdn2d.cu:33-204).  f: fp32 [fh,fw] (separable filters are expanded by the
 * Python wrapper).  x/y element strides in (N,C,H,W) order. */
int n3d_upfirdn2d(const void* x, const float* f, void* y, int dtype, int N, int C, int H, int W,
                  const int64_t x_strides[4], const int64_t y_strides[4], int fh, int fw, int upx, int upy,
                  int downx, int downy, int padx0, int padx1, int pady0, int pady1, int flip, float gain,
                  int outH, int outW, void* stream);

/* bias -> FIR upsample -> lrelu*gain/clamp -> FIR downsample   -- replaces filtered_lrelu_plugin.filtered_lrelu
 * (filtered_lrelu.cpp:20-213), forward only, no sign tensor.  x [N,C,H,W] contiguous, y [N,C,outH,outW] contiguous,
 * fu [fuh,fuw] / fd [fdh,fdw] fp32 2-D filters.  tmp: caller-provided fp32 scratch of N*C*upH*upW floats where
 * upH = H*up + pady0 + pady1 - fuh + 1 (same for W). */
int n3d_filtered_lrelu(const void* x, const float* fu, const float* fd, const void* b, void* y, float* tmp, int dtype,
                       int N, int C, int H, int W, int fuh, int fuw, int fdh, int fdw, int up, int down,
                       int padx0, int padx1, int pady0, int pady1, float gain, float slope, float clamp, int flip,
                       int outH, int outW, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Generator engine: fused building blocks used by TriPlaneGenerator.synthesis (replace the ATen/cuDNN calls the
 * reference makes from networks_stylegan2.py / networks_stylegan2_styleunet.py / superresolution.py).
 * ---------------------------------------------------------------------------------------------------------- */

/* All style vectors of all modulated layers in one launch (FullyConnectedLayer affine, networks_stylegan2.py:303,315
 * and ToRGB's weight_gain :354).  Row r of the concatenated affine matrix belongs to input channel i of some layer:
 *   styles[row_ooff[r] + n * row_cin[r]] = (dot(ws[n, widx[r], :], A[r, :]) / sqrt(wdim) + b[r]) * scale[r]
 * so that every layer owns a dense [N, Cin] block (row_ooff[r] = layer_base * N + i). */
int n3d_styles(const float* ws, int N, int num_ws, int wdim, const float* affine_w, const float* affine_b,
               const int32_t* row_widx, const float* row_scale, const int64_t* row_ooff, const int32_t* row_cin,
               float* styles, int rows, void* stream);

/* Demodulation coefficients of all layers in one launch (networks_stylegan2.py:65).  Row r = output channel o of a layer:
 *   dcoef[row_ooff[r] + n*row_cout[r]] = rsqrt(sum_i styles[row_soff[r] + n*row_cin[r] + i]^2 * wsq[row_woff[r] + i] + 1e-8),
 * wsq[o,i] = sum_k W[o,i,k]^2 (dense [N, Cout] block per layer). */
int n3d_demod(const float* styles, const float* wsq, const int64_t* row_woff, const int32_t* row_cin,
              const int64_t* row_soff, const int64_t* row_ooff, const int32_t* row_cout, float* dcoef, int rows, int N,
              void* stream);

typedef struct {
    int8_t dy, dx;        /* input pixel offset of this tap relative to the output-tile pixel */
    int16_t img_off;      /* selects the input "image" group: image = n + img_off * a_img_mul (parity sub-image of stride-2 convs) */
    int32_t wtap;         /* index of the [Cout, Cin] weight slab for this tap */
} N3DConvTap;

/* Split output of a conv / epilogue.  hi and lo (and style, where the epilogue entry points read it) must be 16-byte aligned. */
typedef struct {
    void* hi;             /* bf16 [.., cstride] or NULL */
    void* lo;
    const float* style;   /* [N, Cout] multiplier applied before the split (next layer's modulation) or NULL */
    int32_t cstride;      /* channel stride of the destination (allows writing into a concat buffer) */
    int32_t coff;         /* channel offset in the destination */
    int32_t f16;          /* 0 (default): split bf16 (hi, lo).  1: fp16 single -- hi is fp16 [.., cstride] holding the value rounded to
                             fp16 (the reference's `.to(float16)` of an SR activation), lo is not read.  Any other value ->
                             N3D_ERR_INVALID_ARG. */
} N3DSplitOut;

/* Optional ToRGB layer (networks_stylegan2.py:353-357) fused into the epilogue of the convolution that produces its input,
 * for image widths <= 4 (the super-resolution blocks): rgb[n,c,pixel] (+)= clamp(sum_o v[n,pixel,o] * style[n,o] * weight[c,o] + bias[c]).
 * Requires all Cout channels of a pixel in one tile (Cout <= 256) and TN == 1 tiles (resolution >= 16). out == NULL disables it. */
typedef struct {
    float* out;            /* fp32 image, NHWC [N,OH,OW,channels] or NCHW */
    const float* weight;   /* [channels, Cout] fp32 */
    const float* style;    /* [N, Cout] fp32 (ToRGB affine output, already multiplied by 1/sqrt(Cout)) */
    const float* bias;     /* [channels] */
    float clamp;           /* < 0 = none */
    int32_t channels, nchw, accumulate;
} N3DFusedRgb;

/* One implicit-GEMM convolution on wgmma tensor cores (bf16 hi/lo operands, 3 products, fp32 accumulate in registers):
 *   acc[n, y, x, o] = sum_taps sum_i A[n + tap.img_off*a_img_mul, y + tap.dy, x + tap.dx, i] * Wp[tap.wtap, o, i]
 * over an M-space of N x MH x MW "tile pixels"; out-of-range A reads are zero (this is the conv padding).
 * Epilogue (mode 0): v = acc * dcoef[n,o] + noise[oy,ox] + bias[o]; v = lrelu_slope(v) * gain; clamp; then any of
 *   out[k].hi/lo <- split_bf16(v * out[k].style[n,o]),  out_f32 <- v (optionally += existing, NHWC or NCHW).
 * Epilogue (mode 1): out_f32 <- acc (raw), used by the transposed-conv parity classes and by split-K.
 * Split-K (splits > 1): for launches with a handful of tiles and a long K loop (the 4^2 / 8^2 layers: one 128-row tile, K = 9 * 512)
 * the taps x channel-chunks are cut into `splits` slices that run as independent work items; deterministic (no atomics).
 * Output pixel of tile pixel (y, x) is (y*oy_mul + oy_off, x*ox_mul + ox_off) in an OH x OW image.
 * Alignment: a_hi, w_hi, out_f32 and every out[k].hi / lo must be 16-byte aligned (else N3D_ERR_INVALID_ARG); split_stride is a
 * multiple of 4.  f32_accumulate cannot be combined with split outputs (N3D_ERR_INVALID_ARG). */
typedef struct {
    const void* a_hi; const void* a_lo;      /* bf16 NHWC [NI, AH, AW, Cin] */
    int32_t NI, AH, AW, Cin;
    const void* w_hi; const void* w_lo;      /* bf16 [T, Cout, Cin] */
    int32_t T, Cout;
    int32_t N, MH, MW;                       /* M-space */
    int32_t a_img_mul;                       /* image coordinate = n + tap.img_off * a_img_mul (parity-major sub-images: = N) */
    int32_t ntaps; N3DConvTap taps[9];
    int32_t nprod;                           /* 3 = hi*hi + hi*lo + lo*hi (fp32-grade), 1 = hi*hi only */
    int32_t mode;
    const float* dcoef;                      /* [N, Cout] or NULL */
    const float* bias;                       /* [Cout] or NULL */
    const float* noise;                      /* [OH, OW] (already multiplied by noise_strength) or NULL */
    int64_t noise_nstride;                   /* 0 = one noise map shared by the batch ('const'), OH*OW = per-sample ('random') */
    float gain, slope, clamp;                /* slope 1 = linear; clamp < 0 = none */
    N3DSplitOut out[2];
    float* out_f32; int32_t f32_cstride, f32_coff, f32_nchw, f32_accumulate;
    int32_t oy_mul, oy_off, ox_mul, ox_off, OH, OW;
    N3DFusedRgb rgb;
    int32_t splits;                          /* > 1: split-K (mode 1 only): K slice s of every tile writes its raw partial sums to */
    int64_t split_stride;                    /*      out_f32 + s * split_stride (elements); reduce with n3d_splitk_epilogue */
    int32_t f16;                             /* 0 (default): bf16 operands as above.  1: fp16 operands -- a_hi fp16 NHWC, w_hi fp16
                                                [T, Cout, Cin], nprod must be 1 (a_lo / w_lo are not read): one wgmma...f32.f16.f16 per
                                                k16 step, fp32 accumulate, as the reference's fp16 SR convolutions on CUDA
                                                (networks_stylegan2.py:54-79 with x.dtype == float16).  Every used out[k] must then be
                                                fp16 single (out[k].f16 = 1), and with f16 = 0 none may be. */
} N3DConvGemm;

int n3d_conv_gemm(const N3DConvGemm* p, void* stream);

/* Stride-2 transposed 3x3 convolution (the first half of every up-sampling conv: conv_transpose2d(stride 2),
 * conv2d_resample.py:114-127) as ONE launch of the same kernel: the four output-parity classes
 *   out[2p+a, 2q+b] = sum_{ky = a (mod 2), kx = b (mod 2)} W[ky,kx] x[p - (ky-a)/2, q - (kx-b)/2]
 * are four sub-problems (4/2/2/1 taps) scheduled together.  p->MH, p->MW = INPUT height / width, p->T must be 9; the raw fp32
 * NHWC result [N, 2H+1, 2W+1, Cout] is written to p->out_f32 (f32_cstride / f32_coff honoured); taps, offsets, OH/OW, mode and
 * the epilogue fields of the descriptor are ignored (follow with n3d_fir_up_epilogue). */
int n3d_conv_transposed_gemm(const N3DConvGemm* p, void* stream);

/* Weight gradient of a convolution as one launch over all groups and taps (plus a reduction launch when splits > 1):
 *   dw[g, t, m, n] = sum_{k < K} A[a_row[t] + g*M + m, k + a_off[t]] * B[b_row[t] + g*N + n, k + b_off[t]]
 * A (output gradient) and B (layer input) are channel-major split bf16 (hi, lo), one row per channel, laid out by
 * n3d_wgrad_operand; a tap is a column offset (a multiple of 8: TMA boxes start on 16-byte boundaries) plus a row offset (which
 * selects a copy of the operand shifted by a few columns), and reads outside [0, a_cols) / [0, b_cols) are zero.  bf16x3 products, fp32
 * accumulate.  K (a multiple of 64) is cut into `splits` slices (1 <= splits <= K / 64): slice s writes partial + s * G*T*M*N and a
 * second kernel sums the slices in order into dw (no atomics: bit-identical from run to run).  N a multiple of 8.  Operands, partial
 * and dw 16-byte aligned; lda, ldb multiples of 8. */
typedef struct {
    const void* a_hi; const void* a_lo;      /* bf16 [a_rows, lda] */
    int32_t a_rows; int64_t a_cols, lda;
    const void* b_hi; const void* b_lo;      /* bf16 [b_rows, ldb] */
    int32_t b_rows; int64_t b_cols, ldb;
    int32_t G, M, N, T;                      /* groups, rows of dw (output channels), columns (input channels), taps <= 9 */
    int64_t K;
    int64_t a_off[9], b_off[9];              /* per-tap column offsets: multiples of 8, may be negative */
    int32_t a_row[9], b_row[9];              /* per-tap row offsets (>= 0, row + G*M <= a_rows, row + G*N <= b_rows) */
    int32_t splits;
    float* partial;                          /* fp32 [splits, G, T, M, N] (splits > 1) */
    float* dw;                               /* fp32 [G, T, M, N] */
} N3DConvWgrad;

int n3d_conv_wgrad(const N3DConvWgrad* p, void* stream);

/* Operand of n3d_conv_wgrad from an fp32 tensor x [N, C, H, W] with element strides x_strides (n, c, y, x):
 *   hi/lo[c * ld + j - shift] = split_bf16(x[n, c, s*(py - pt) + par / s, s*(px - pl) + par % s]),  j = ((par * N + n) * PH + py) * PW + px
 * for par < s*s (s = 1, or 2 = parity sub-images of a stride-2 tap); every other column of [0, ld) is 0 (source pixel outside x,
 * j outside [0, s*s*N*PH*PW)).  shift moves the grid `shift` columns left (a horizontal tap shift).  ld a multiple of 8; hi / lo
 * 16-byte aligned. */
int n3d_wgrad_operand(const float* x, const int64_t x_strides[4], int N, int C, int H, int W, int s, int pt, int pl, int PH, int PW,
                      int shift, int64_t ld, void* hi, void* lo, void* stream);

/* fp32 NHWC -> split bf16 NHWC with optional per-(n,c) modulation: out = split(x[n,y,x,c] * style[n,c]).
 * Alignment: x and style 16-byte aligned (float4 loads), hi and lo 8-byte aligned (4-channel stores); C, out_cstride and out_coff
 * multiples of 4; else N3D_ERR_INVALID_ARG. */
int n3d_modulate_split(const float* x, int64_t npix_per_img, int N, int C, const float* style, void* hi, void* lo,
                       int out_cstride, int out_coff, void* stream);
/* n3d_modulate_split with an fp16 single output: out = fp16(x[n,y,x,c] * style[n,c]) -- the first fp16 SR block's input at a
 * 128^2 rendering, x.to(float16) then the modulation (networks_stylegan2.py:557, 73).  Same argument checks, out in place of hi / lo. */
int n3d_modulate_f16(const float* x, int64_t npix_per_img, int N, int C, const float* style, void* out, int out_cstride, int out_coff,
                     void* stream);

/* Second half of an up-sampling modulated conv (conv2d_resample.py:114-131 + networks_stylegan2.py:320-329):
 * raw [(2H+1),(2W+1)] transposed-conv output (fp32 NHWC) -> 4x4 FIR [1,3,3,1]^2/64 * 4, pad 1 -> [2H,2W], then the
 * same epilogue as n3d_conv_gemm mode 0 (requires gain > 0 and 0 <= slope <= 1: lrelu / linear).
 * Alignment (this and n3d_splitk_epilogue): raw / partial, dcoef, bias, out_f32 and each used out[k].hi / lo / style must be 16-byte
 * aligned; f32_cstride, f32_coff, out[k].cstride and out[k].coff are multiples of 4. */
int n3d_fir_up_epilogue(const float* raw, int N, int H2, int W2, int C, const float* dcoef, const float* bias,
                        const float* noise, int64_t noise_nstride, float gain, float slope, float clamp,
                        const N3DSplitOut out[2], float* out_f32, int f32_cstride, int f32_coff, void* stream);

/* Second pass of a split-K convolution: y = sum_s partial[s] (fixed order) followed by the mode-0 epilogue of n3d_conv_gemm
 * (demod, noise, bias, lrelu * gain, clamp, modulated split-bf16 copies, fp32 copy).  partial: fp32 NHWC [S][N,H,W,C]. */
int n3d_splitk_epilogue(const float* partial, int S, int64_t split_stride, int N, int H, int W, int C, const float* dcoef,
                        const float* bias, const float* noise, int64_t noise_nstride, float gain, float slope, float clamp,
                        const N3DSplitOut out[2], float* out_f32, int f32_cstride, int f32_coff, void* stream);

/* First half of a down-sampling conv (conv2d_resample.py:108-111): fp32 NHWC [H,W] -> FIR pad (2,2,2,2) -> [(H+1),(W+1)]
 * -> split bf16, de-interleaved by pixel parity into 4 sub-images [4, N, SH, SW, C] (parity (y&1)*2 + (x&1), pixel
 * (y>>1, x>>1)), SH = (H+2)/2, so that the stride-2 conv becomes 9 unit-stride taps.
 * Alignment: x 16-byte aligned (float4 loads), hi and lo 8-byte aligned (4-channel stores); C a multiple of 4, H and W even; else
 * N3D_ERR_INVALID_ARG. */
int n3d_fir_down_split(const float* x, int N, int H, int W, int C, void* hi, void* lo, void* stream);

/* upfirdn2d.upsample2d on an fp32 NHWC image (up 2, pad (2,1), gain 4; networks_stylegan2.py:577); y is NHWC, or NCHW
 * when y_nchw != 0 (used for the final image).  Any alignment: 4 channels per thread (float4) when C % 4 == 0 and x and an NHWC y
 * are 16-byte aligned, else one channel per thread. */
int n3d_upsample2d_nhwc(const float* x, int N, int H, int W, int C, float* y, int y_nchw, void* stream);
/* upfirdn2d.downsample2d on an fp32 NHWC image (pad (1,1), down 2; networks_stylegan2_styleunet.py:109). */
int n3d_downsample2d_nhwc(const float* x, int N, int H, int W, int C, float* y, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Mesh path: FLAME neural-texture rasterization into the orthographic views (triplane_next3d.py:190-230).
 * ---------------------------------------------------------------------------------------------------------- */

/* View transform of vertices / landmarks for the 4 rendering views (triplane_next3d.py:194-205; rotation matrices
 * are supplied by the caller, [4,3,3] fp32, computed with the reference's fp32 sin/cos):
 *   out[n, view, i, :] = flipY(p) @ R_view + shift, * scale, negate y,z; z += zoff.  Also applies the rasterizer
 * wrapper's x,y negation (renderer.py:403) when ndc_flip != 0. */
int n3d_transform_points(const float* pts, int N, int P, const float* rot, int nviews, float zoff, int ndc_flip,
                         float* out, void* stream);

/* pytorch3d-semantics rasterizer (SURVEY.md Appendix C; oracle/oracle_c.c is the bit-exact CPU statement) -- replaces
 * pytorch3d.renderer.mesh.rasterize_meshes as called at volumetric_rendering/renderer.py:414-424 (blur 0, 1 face/pixel,
 * cull_backfaces, no perspective correction).  verts [NM, V, 3] NDC fp32, faces [F,3] int32 (shared by all images)
 * -> pix_to_face [NM,H,W] int32 (face id or -1), bary [NM,H,W,3] fp32 (-1 where empty).
 * workspace: caller-provided, 16-byte aligned, NM * F * 16 floats (per-face setup records shared by all pixel bins). */
int n3d_rasterize(const float* verts, const int32_t* faces, int NM, int V, int F, int H, int W, int32_t* pix_to_face,
                  float* bary, float* workspace, void* stream);

/* Texture lookup for the 4 rendered views of each sample (triplane_next3d.py:211-228, renderer.py:425-437):
 *   uv = sum_k bary_k * face_uv[f,k,:] (0 where nothing is visible); value = bilinear(texture[n], uv) (grid_sample, zeros
 *   padding, align_corners False); alpha = bilinear(eye_mask, uv) * visible.
 * pix_to_face / bary are [N*4,H,W(,3)] with image index n*4 + view; face_uv [F,3,2]; texture NHWC [N,TH,TW,C<=32];
 * eye_mask [MH,MW].  Outputs (plane-major): tex_planes [3,N,H,W,C] = (view0, view1 + view2, view3) and alpha [3,N,H,W] =
 * (view0, view1, view3) -- the reference's `alpha[1] | alpha[1]` quirk (:226) means view 2's alpha is never used. */
int n3d_uv_sample(const int32_t* pix_to_face, const float* bary, const float* face_uv, const float* texture,
                  const float* eye_mask, int N, int H, int W, int TH, int TW, int C, int MH, int MW,
                  float* tex_planes, float* alpha, void* stream);
/* n3d_uv_sample for several images per texture: image n (of N) reads texture[n / views], so texture is [N / views,TH,TW,C];
 * every other argument and output is per image, as above.  views = 1 is n3d_uv_sample.  views < 1 or N not a multiple of
 * views -> N3D_ERR_INVALID_ARG before any launch. */
int n3d_uv_sample_views(const int32_t* pix_to_face, const float* bary, const float* face_uv, const float* texture,
                        const float* eye_mask, int N, int views, int H, int W, int TH, int TW, int C, int MH, int MW,
                        float* tex_planes, float* alpha, void* stream);

/* fill_mouth (renderer.py:583-602): alpha [NI,H,W] in place; cv2.floodFill from (0,0) with fixed range [seed, seed+254]
 * on alpha*255, then alpha += 1 - (filled/127.5 - 1), clipped to [0,1].  H*(W+4) <= 200 KB (512x396 at most).
 * One CTA per image; the sweeps repeat until the fill has converged, however winding the region. */
int n3d_fill_mouth(float* alpha, int NI, int H, int W, void* stream);
/* n3d_fill_mouth, after which images [bin0, bin1) are binarized, alpha = (alpha != 0) (a NaN gives 1): what the reference
 * does to the side plane's alpha (triplane_next3d.py:226).  0 <= bin0 <= bin1 <= NI; bin0 = bin1 is n3d_fill_mouth. */
int n3d_fill_mouth_binarize(float* alpha, int NI, int H, int W, int bin0, int bin1, void* stream);

/* gen_mouth_mask (triplane_next3d.py:330-344) on device: lm2d [N,68,2] -> boxes [N,4] int32 (y0,y1,x0,x1). */
int n3d_mouth_box(const float* lm2d, int N, int32_t* boxes, void* stream);

/* Antialiased bilinear resize (ATen _upsample_bilinear2d_aa, SURVEY.md A.10) between per-sample boxes of NHWC images --
 * replaces F.interpolate(..., antialias=True) at triplane_next3d.py:152,161 and superresolution.py:282-286:
 *   dst[n, ty0:ty1, tx0:tx1, :] = resize(src[n, sy0:sy1, sx0:sx1, :]) to (ty1-ty0, tx1-tx0).
 * src_box / dst_box: device int32 [N,4] = (y0,y1,x0,x1) or NULL (= whole image); destination pixels outside the box are
 * left untouched.  dst may be NULL when only the split output is wanted; hi/lo (optional): split_bf16(value * style[n,c]). */
int n3d_resize_aa(const float* src, int N, int SH, int SW, int C, const int32_t* src_box, float* dst, int DH, int DW,
                  const int32_t* dst_box, const float* style, void* hi, void* lo, void* stream);
/* n3d_resize_aa with only an fp16 single output: out[n, y, x, c] = fp16(resize(src)[n, y, x, c] * style[n, c]) (style may be NULL) --
 * the SR input features resized to 128^2 (superresolution.py:282-286), then x.to(float16) and the first fp16 block's modulation. */
int n3d_resize_aa_f16(const float* src, int N, int SH, int SW, int C, const int32_t* src_box, int DH, int DW, const int32_t* dst_box,
                      const float* style, void* out, void* stream);

/* planes[n,p,y,x,c] = tex[n,p,y,x,c] * alpha[n,p,y,x] + static[n,y,x,p*32+c] * (1 - alpha)  (triplane_next3d.py:171-174);
 * tex for plane 0 = blended_front NHWC [N,H,W,32] (neural-blending output), planes 1,2 = tex_planes[1:] (plane-major
 * [3,N,H,W,32]), alpha [3,N,H,W], static_planes NHWC [N,H,W,96]; planes out channels-last [N,3,H,W,32].
 * Alignment: blended_front, tex_planes, static_planes and planes 16-byte aligned (float4 loads / stores), else N3D_ERR_INVALID_ARG. */
int n3d_blend_planes(const float* blended_front, const float* tex_planes, const float* alpha, const float* static_planes,
                     int N, int H, int W, float* planes, void* stream);
/* n3d_blend_planes for several images per static plane set: image n (of N) reads static_planes[n / views], so static_planes is
 * NHWC [N / views,H,W,96]; every other argument and output is per image.  views = 1 is n3d_blend_planes.  views < 1 or N not a
 * multiple of views -> N3D_ERR_INVALID_ARG before any launch. */
int n3d_blend_planes_views(const float* blended_front, const float* tex_planes, const float* alpha, const float* static_planes,
                           int N, int views, int H, int W, float* planes, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Volume renderer: ray generation + stratified sampling + tri-plane fetch + MLP decode + importance resampling +
 * sort-merge + alpha compositing in one kernel per ray batch (ray_sampler.py:24-63, renderer.py:95-268,
 * triplane_next3d.py:348-371, ray_marcher.py:27-66).
 * ---------------------------------------------------------------------------------------------------------- */
/* Alignment: planes must be 32-byte aligned (each texel's 32 channels are read as 256-bit loads), else N3D_ERR_INVALID_ARG. */
typedef struct {
    const float* planes;       /* [N,3,PH,PW,32] channels-last fp32, 32-byte aligned */
    int32_t N, PH, PW;
    const float* cam2world;    /* [N,16] */
    const float* intrinsics;   /* [N,9]  */
    int32_t res;               /* rays = res*res per sample */
    int32_t depth_coarse, depth_fine;  /* samples per pass: 4 .. 192 coarse, 0 (coarse only) .. 192 fine; above 192 -> N3D_ERR_UNSUPPORTED */
    float ray_start, ray_end, box_warp;
    const float* u_coarse;     /* [N, M, Dc] injected uniforms or NULL (= in-kernel counter RNG with `seed`) */
    const float* u_fine;       /* [N*M, Df] or NULL */
    uint64_t seed;
    const uint64_t* seed_ptr;  /* optional device counter added to `seed` (lets a captured CUDA graph draw fresh noise per replay) */
    const float* w0; const float* b0;   /* decoder.net.0: [64,32] (already * 1/sqrt(32)), [64] */
    const float* w1; const float* b1;   /* decoder.net.2: [33,64] (already * 1/sqrt(64)), [33] */
    float* rgb;                /* [N, M, 32] */
    float* depth;              /* [N, M] (unclamped) */
    float* wsum;               /* [N, M] */
    float* depth_minmax;       /* [2] device: running min / max of all sample depths (init +inf / -inf by caller); [N, 2] when
                                  depth_range_per_image = 1 */
    int32_t white_back;
    int32_t views;             /* camera views per plane set: 0 or 1 = image n reads plane set n; V >= 2 = image n reads plane set
                                  n / V, so `planes` holds N / V sets (N a multiple of V).  Cameras, uniforms, outputs and depth_minmax
                                  stay per image. */
    int32_t depth_range_per_image;  /* 0: depth_minmax [2] covers the whole launch (ray_marcher.py:54 on a batch).  1: depth_minmax
                                  [N, 2], pair n reduced over image n's samples only (each pair initialised to +inf / -inf by the
                                  caller; with views = V the pair is the image's, not the plane set's), as when every image is rendered
                                  by a launch of its own.  Any other value -> N3D_ERR_INVALID_ARG. */
    double ray_span;           /* ray_end - ray_start as the caller holds them (double), or 0 = the difference of the float fields.  The
                                  coarse jitter spacing is ray_span / (depth_coarse - 1) rounded to float, as renderer.py:204 forms it
                                  from Python floats; the float endpoints are each off by up to half an ulp, 1.7e-4 of a 1e-3 interval. */
} N3DRender;

int n3d_render_rays(const N3DRender* p, void* stream);
/* n3d_render_rays plus surface normals (ImportanceRenderer.normal_forward + MipRayMarcher2 with return_normal,
 * renderer.py:271-355, ray_marcher.py:32-33,61-64): writes rgb / depth / wsum / depth_minmax exactly as n3d_render_rays does and
 * normal [N, M, 3] = the unit-length composite of n = -d sigma_raw / d x (world space) over the same samples and final weights.
 * workspace: device float32 buffer of N * M * (2D - 1) floats, D = depth_coarse + depth_fine (depth_coarse when depth_fine = 0);
 * it holds each ray's sorted sample depths and final weights between the renderer and the normal kernel.  Same argument checks
 * and sample-count limits as n3d_render_rays.  Two kernel launches. */
int n3d_render_rays_normals(const N3DRender* p, float* normal, float* workspace, void* stream);
/* Diagnostics: the normal pass of n3d_render_rays_normals alone, over the samples an earlier n3d_render_rays_normals call with the
 * same p left in `workspace`.  tools/bench_render.py --normals times it (DESIGN.md section 3.2a). */
int n3d_render_normals_pass(const N3DRender* p, const float* workspace, float* normal, void* stream);
/* Diagnostics: micro-kernels that measure the hard per-SM limits of the renderer's formulation on the workload described by p
 * (only planes / cameras / res / depth_* / ray_* / box_warp are read; nothing is written but sink[0], which may be NULL):
 * kind 0 = the tri-plane gather alone (rays, depths, 12 taps per sample, 256-bit loads, weighted sum, bf16 split, shared-memory
 * tile) on all warps; kind 1 = the decoder's activations alone (192 MUFU operations per sample).  bench.py times them next to
 * n3d_render_rays to report how far the fused kernel is from what a per-sample gather + MLP can reach (DESIGN.md section 3.2).
 * Up to 96 samples per pass (the 16- and 32-lane layouts); `views` is honoured and checked as in n3d_render_rays. */
int n3d_render_floor(const N3DRender* p, int kind, float* sink, void* stream);
/* composite depth clamp to the batch-global depth range (ray_marcher.py:53-54). */
int n3d_depth_clamp(float* depth, int64_t n, const float* depth_minmax, void* stream);
/* the same clamp per image (depth_range_per_image = 1): depth [N, per_image] elements of image n clamped to depth_minmax[n] of
 * depth_minmax [N, 2].  N >= 0, per_image >= 0, non-null pointers; otherwise N3D_ERR_INVALID_ARG. */
int n3d_depth_clamp_images(float* depth, int N, int64_t per_image, const float* depth_minmax, void* stream);
/* run_model only (TriPlaneGenerator.sample, triplane_next3d.py:276): coords [N,P,3] -> sigma [N,P], rgb [N,P,32] (or NULL).
 * planes must be 32-byte aligned (256-bit texel loads) and rgb 8-byte aligned (float2 stores), else N3D_ERR_INVALID_ARG. */
int n3d_sample_points(const float* planes, int N, int PH, int PW, const float* coords, int64_t P, float box_warp,
                      const float* w0, const float* b0, const float* w1, const float* b1, float* sigma, float* rgb,
                      void* stream);

/* Shape-extraction grid (gen_samples_next3d.py:80-102, 208-238): sigma at the voxel centres of create_samples(N = grid_n,
 * cube_length) for the flat indices head .. head+count-1, coordinates generated in the kernel with the script's own float32
 * operations (no [N^3,3] coordinate tensor), written into sigma_grid [grid_n]^3 at the position the script's
 * flip(dims=[0]) + border trim leaves them; voxels inside the trimmed border (width `pad`, the script's int(30 * N / 256))
 * receive pad_value and are not decoded.  pad = 0: plain flip.  Planes of ONE sample [3,PH,PW,32], 32-byte aligned (else
 * N3D_ERR_INVALID_ARG). */
int n3d_sample_grid(const float* planes, int PH, int PW, int grid_n, float cube_length, float box_warp, int64_t head, int64_t count,
                    int pad, float pad_value, const float* w0, const float* b0, const float* w1, const float* b1, float* sigma_grid,
                    void* stream);

/* MappingNetwork + truncation in one launch (networks_stylegan2.py:233-268, called through triplane_next3d.py:111-115 with
 * c[:, :25] * c_scale): z [N,512], c [N,25] -> ws [N,num_ws,512].  embed / fc0 / fc1 are the raw parameters of
 * `backbone.mapping` (weight [out,in], bias [out]); their runtime gains (1/sqrt(in), lr_multiplier 0.01) are applied inside.
 * truncation_cutoff < 0 = all layers; w_avg may be NULL when truncation_psi == 1. */
int n3d_mapping(const float* z, const float* c, int N, float c_scale, const float* embed_w, const float* embed_b, const float* fc0_w,
                const float* fc0_b, const float* fc1_w, const float* fc1_b, const float* w_avg, float truncation_psi,
                int truncation_cutoff, int num_ws, float* ws, void* stream);

/* out[f, :] = sum_k B[f, k] * Y[k, :]  (B [F,K], Y [K,D], fp32): the frame drivers' latent interpolation (B = the cubic-spline
 * basis of gen_videos_next3d.py:106-117 evaluated once on the host) and camera smoothing (reenact_avatar_next3d.py:159) on the
 * device. */
int n3d_interp_rows(const float* B, const float* Y, int F, int K, int64_t D, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Host-side input parsers (no device work; SURVEY.md section 8 row f3): what the inference scripts do per frame in Python.
 * ---------------------------------------------------------------------------------------------------------- */

/* Vertex positions of a Wavefront .obj text (gen_samples_next3d.py:165-174: every line with line[:2] == "v ", tokens after the
 * first converted with float(), all numbers flattened and reshaped to (-1, 3), then .float()).  text need not be NUL-terminated.
 * Writes up to max_vertices * 3 floats; *n_vertices receives the count (also when it exceeds max_vertices -> INVALID_ARG, so a
 * caller can size the buffer with max_vertices = 0 first). */
int n3d_parse_obj_vertices(const char* text, int64_t len, float* xyz, int64_t max_vertices, int64_t* n_vertices);

/* Whitespace-separated table of numbers with '#' comments, the subset of np.loadtxt the scripts use for *_kpt2d.txt
 * (gen_samples_next3d.py:176-177): float64 parse, float32 store; every non-empty row must have *n_cols columns. */
int n3d_parse_float_table(const char* text, int64_t len, float* values, int64_t max_values, int64_t* n_values, int64_t* n_cols);

/* ------------------------------------------------------------------------------------------------------------
 * H.264 encoder (next3d_b200/video.py; DESIGN.md section 3): Constrained Baseline (profile_idc 66), 8-bit 4:2:0 BT.601 limited
 * range, CAVLC, one slice per macroblock row, IDR frames of I_16x16 macroblocks, P frames of P_L0_16x16 / P_Skip predicted from
 * the previous frame.  Two streams share the buffers and the argument checks:
 *   constant QP (n3d_h264_encode): integer-pel motion, deblocking disabled (so the reconstruction is the decoder's output);
 *   rate-controlled (n3d_h264_encode_rc): one QP per picture chosen on the device, quarter-sample motion, in-loop deblocking.
 * In both, recon receives the decoder's output picture, which the caller passes back as the next P frame's ref.  The caller
 * owns the reconstruction buffers (and the controller state); the encoder keeps nothing between calls.  The SPS / PPS are
 * written by the caller (next3d_b200.video.sps / pps: log2_max_frame_num 4, pic_order_cnt_type 2, pic_init_qp = qp for the
 * constant-QP stream and 26 for the rate-controlled one).
 * ---------------------------------------------------------------------------------------------------------- */

/* Host only.  Buffer sizes in bytes for width x height frames: plane_bytes = one padded I420 picture (width and height rounded
 * up to multiples of 16; Y, then Cb, then Cr), scratch_bytes = per-macroblock state, slice_bytes = one bounded slot per
 * macroblock row, sample_bytes = capacity of one encoded frame.  The slot bound is derived from the syntax written (27 residual
 * blocks of at most 641 bits plus a 128-bit macroblock header, emulation prevention included); the Annex A limit of 3200 bits
 * per macroblock is not enforced (it can be exceeded only at very low QP on noise).  N3D_ERR_INVALID_ARG for odd or
 * non-positive sizes and frames above level 6.2 (139264 macroblocks, at most 1055 per side). */
int n3d_h264_buffer_sizes(int width, int height, int64_t* plane_bytes, int64_t* scratch_bytes, int64_t* slice_bytes,
                          int64_t* sample_bytes);

/* Encode one frame.  rgb: device uint8 [height, width, 3] contiguous.  qp 0..51.  idr != 0: IDR picture (ref unused, may be
 * NULL); else a P picture predicted from ref (the previous frame's recon, plane_bytes, != recon).  frame_num: 0..15 (frames
 * since the last IDR, mod 16); idr_pic_id 0..65535 (must differ between consecutive IDR pictures).  cur (plane_bytes), scratch
 * and slices are work space; recon (plane_bytes) receives the reconstruction.  sample (sample_bytes) receives the access unit as
 * length-prefixed NAL units (4-byte big-endian lengths, one slice per macroblock row) and *sample_len (device int64) its size,
 * or -1 if a slice exceeded its slot (the slot is never written past).  No host synchronisation. */
int n3d_h264_encode(const uint8_t* rgb, int width, int height, int qp, int idr, int frame_num, int idr_pic_id, uint8_t* cur,
                    const uint8_t* ref, uint8_t* recon, void* scratch, uint8_t* slices, uint8_t* sample, int64_t* sample_len,
                    void* stream);

/* Rate-controlled stream: the same encoder with one QP per picture chosen on the device (no host synchronisation), quarter-sample
 * motion vectors and in-loop deblocking across slice boundaries (the deblocked picture is recon and the next P frame's
 * reference).  Its PPS has pic_init_qp 26 (next3d_b200.video.pps(26)); each slice carries slice_qp_delta = QP - 26.
 * The controller state is N3D_H264_RC_STATE_BYTES of caller-owned device memory (8-byte aligned), written by n3d_h264_rc_init and
 * updated on the stream after every n3d_h264_encode_rc from *sample_len: a one-second leaky bucket in integer arithmetic, QP
 * changing by at most 2 between consecutive P frames and kept across IDR frames, clamped to qp_min..qp_max (equal bounds pin it). */
#define N3D_H264_RC_STATE_BYTES 128

/* Stream-ordered: writes the state for width x height frames at bits_per_second (1..2^32-1) and fps_num / fps_den frames/s
 * (each 1..2^20), QP bounds 0 <= qp_min <= qp_max <= 51; the first QP follows from the bits per pixel.  N3D_ERR_INVALID_ARG
 * for a null state, the sizes n3d_h264_buffer_sizes refuses, or values out of range. */
int n3d_h264_rc_init(void* state, int width, int height, int64_t bits_per_second, int fps_num, int fps_den, int qp_min, int qp_max,
                     void* stream);

/* n3d_h264_encode with the controller state (initialised by n3d_h264_rc_init for the same size) in place of qp; the same
 * buffers and argument checks.  No host synchronisation. */
int n3d_h264_encode_rc(const uint8_t* rgb, int width, int height, void* state, int idr, int frame_num, int idr_pic_id, uint8_t* cur,
                       const uint8_t* ref, uint8_t* recon, void* scratch, uint8_t* slices, uint8_t* sample, int64_t* sample_len,
                       void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * PNG encoder (next3d_b200/png.py; DESIGN.md section 3.6): n uint8 RGB images [height, width, 3] -> n complete PNG files
 * (signature, IHDR 8-bit RGB without interlace, one IDAT chunk, IEND).  A file's bytes are a function of its image alone: they
 * do not depend on n, the stream or the device.  The numpy restatement is tests/png_oracle.py.
 * ---------------------------------------------------------------------------------------------------------- */

/* Host only.  scratch_bytes: work space of one n3d_png_encode call of n images; file_bytes: capacity of one file (the size of
 * the image in stored deflate blocks, which no file exceeds).  N3D_ERR_INVALID_ARG for n, height or width < 1, width > 2^24,
 * or an image whose IDAT chunk could exceed 2^31 - 1 bytes. */
int n3d_png_buffer_sizes(int n, int height, int width, int64_t* scratch_bytes, int64_t* file_bytes);

/* Encode n images.  rgb: device uint8 [n, height, width, 3] contiguous; scratch: scratch_bytes (256-byte aligned); files:
 * n * file_bytes, file i at i * file_bytes; *file_lens (device int64 [n]) receives each file's length.  Stream-ordered, no host
 * synchronisation. */
int n3d_png_encode(const uint8_t* rgb, int n, int height, int width, void* scratch, uint8_t* files, int64_t* file_lens,
                   void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Marching cubes (next3d_b200/isosurface.py; DESIGN.md section 3.7): the mesh of the level set of a float32 grid
 * g[a0, a1, a2] of shape [nz, ny, nx] (the layout of n3d_sample_grid and of the .mrc data).  A voxel is inside when g > level;
 * one vertex per grid edge whose endpoints differ, at (x, y, z) = (a2, a1, a0) plus t = (level - s0) / (s1 - s0) along the
 * edge (fp32, IEEE division), in ascending (a0, a1, a2) of the edge's lower endpoint, then its x-, y- and z-edge; triangles cell
 * by cell in ascending (a0, a1, a2), each cell's from its 256-entry table, wound so that the right-hand normal points from the
 * inside toward the outside.  A grid with a dimension below 2 has no cells and an empty mesh.  The result depends on the grid
 * and the level alone.  The numpy restatement is tests/isosurface_oracle.py.
 * ---------------------------------------------------------------------------------------------------------- */

/* Host only.  Workspace of a grid: three int64 per (a0, a1) voxel row and per tile of 4096 rows (O(nz * ny), never O(voxels)).
 * N3D_ERR_INVALID_ARG for a dimension < 1, nz * ny > 2^31 - 4097 or nx > 2^28. */
int n3d_isosurface_workspace_bytes(int nz, int ny, int nx, size_t* bytes);

/* Pass 1: classify every voxel row, scan the rows; counts (device int64 [3]) receives {vertices, triangles, non-finite voxels},
 * and the workspace (8-byte aligned) keeps the rows' offsets for n3d_isosurface_emit.  level must be finite.  Stream-ordered, no
 * host synchronisation. */
int n3d_isosurface_count(const float* grid, int nz, int ny, int nx, float level, void* workspace, int64_t* counts, void* stream);

/* Pass 2, after n3d_isosurface_count of the same grid, level and workspace: verts (device float32 [V, 3]) and faces (device int32
 * [F, 3], vertex indices) of the counted mesh.  The caller checks V and F below 2^31 first.  Stream-ordered. */
int n3d_isosurface_emit(const float* grid, int nz, int ny, int nx, float level, const void* workspace, float* verts, int32_t* faces,
                        void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Vertex colours of a shape mesh (next3d_b200/bake.py; DESIGN.md section 3.8).  Cameras are the renderer's: cam2world [views, 16]
 * row-major and normalised intrinsics [views, 9], as n3d_render_rays reads them; a world point projects to camera depth z (the
 * camera's +z axis) and pixel (u, w) = (xc * width - 0.5, yc * height - 0.5), pixel centres at integers.  Every operation is a
 * rounded fp32 operation without contraction; the numpy restatement is tests/bake_oracle.py.
 * ---------------------------------------------------------------------------------------------------------- */

/* World points world [nv, 3] of mesh vertices verts [nv, 3] in voxel units (x, y, z) = (a2, a1, a0) of the flipped shape grid of
 * create_samples(grid_n, cube): s1 = y + x / R, s0 = (R - 1 - z) + s1 / R, s2 = x, p = s * cube / (R - 1) - cube / 2.  grid_n >= 2,
 * cube finite and positive.  Stream-ordered. */
int n3d_bake_world_points(const float* verts, int64_t nv, int grid_n, float cube, float* world, void* stream);

/* Z-buffer zbuf [views, height, width] (uint64, 8-byte aligned) of the triangles faces [nf, 3] (int32) over world points verts
 * [nv, 3]: each pixel holds the least (depth bits << 32 | triangle id) over the triangles whose edges hold its centre (edges
 * included), depth the perspective-correct camera depth there; ~0 where no triangle covers it.  Triangles with a vertex at z <= near,
 * a vertex index outside [0, nv), zero signed area or non-finite corners are skipped.  The result does not depend on the launch.
 * nv, nf < 2^31; near finite and positive.  Stream-ordered. */
int n3d_mesh_zbuffer(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* cam2world, const float* intrinsics,
                     int views, int height, int width, float near, uint64_t* zbuf, void* stream);

/* colors [nv, 3] (uint8) of the vertices verts [nv, 3] (voxel units) at world points world [nv, 3] (n3d_bake_world_points), on the
 * density grid [grid_n]^3 they were meshed from, from the images [views, 3, height, width] (float32, -1..1) and the z-buffer of
 * n3d_mesh_zbuffer.  In view order, a vertex is visible when z > near, its nearest pixel lies in the image and z <= the pixel's depth
 * + eps (an empty pixel is infinitely deep); its weight is visible * max(0, n . d)^2, n the normalised outward normal -grad sigma
 * (trilinear central differences mapped to world space) and d the unit vector to the camera centre; the colour is the weighted
 * mean of the images' bilinear samples, else (no weight) 2 f - 1 of f = fallback[i * fallback_stride + 0..2], the decoder's colour in
 * the range n3d_sample_points writes (about 0..1; 2 f - 1 is the ray marcher's rescaling, what image_raw shows), as uint8 clamp(c * 127.5 + 128, 0,
 * 255).  visible [views, nv] (uint8 0/1) and weights [views, nv] (float32) receive the per-view values unless NULL.  Stream-ordered. */
int n3d_bake_vertex_colors(const float* verts, const float* world, int64_t nv, const float* grid, int grid_n, const float* cam2world,
                           const float* intrinsics, int views, const float* images, int height, int width, const uint64_t* zbuf,
                           float near, float eps, const float* fallback, int fallback_stride, uint8_t* colors, uint8_t* visible,
                           float* weights, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NEXT3D_B200_H */
