// Memory-bound glue kernels of the generator engine (everything between two tensor-core convolutions that could not be
// folded into a GEMM epilogue).  All tensors NHWC; 128-bit accesses along the channel dimension; grids sized in
// multiples of the SM count.
#include <cstdlib>
#include "common.cuh"
#include <cuda.h>
#include "tc_ptx.cuh"

namespace {
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---------------------------------------------------------------------------------------------- styles / demod
// one warp per (row, n): 512-long dot product with float4 loads
// output layout: every layer owns a dense [N, Cin] block: styles[ooff[r] + n * cin[r]]
__global__ void __launch_bounds__(256) styles_kernel(const float* __restrict__ ws, int N, int num_ws, int wdim,
                                                     const float* __restrict__ A, const float* __restrict__ b,
                                                     const int* __restrict__ widx, const float* __restrict__ scale,
                                                     const int64_t* __restrict__ ooff, const int* __restrict__ cin,
                                                     float* __restrict__ styles, int rows) {
    const int lane = threadIdx.x & 31;
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const float inv = rsqrtf((float)wdim);
    for (int64_t r = warp_global; r < rows; r += nwarps) {
        const float4* a4 = reinterpret_cast<const float4*>(A + r * wdim);
        const int wi = widx[r];
        for (int n = 0; n < N; ++n) {
            const float4* w4 = reinterpret_cast<const float4*>(ws + ((int64_t)n * num_ws + wi) * wdim);
            float acc = 0.f;
            for (int i = lane; i < wdim / 4; i += 32) {
                const float4 a = __ldg(a4 + i), w = __ldg(w4 + i);
                acc += a.x * w.x + a.y * w.y + a.z * w.z + a.w * w.w;
            }
            acc = warp_sum(acc);
            if (lane == 0) styles[ooff[r] + (int64_t)n * cin[r]] = (acc * inv + b[r]) * scale[r];
        }
    }
}

// one warp per output channel row r of some layer: styles of that layer at styles[soff[r] + n*cin[r] + i],
// result at dcoef[ooff[r] + n*cout[r]] (dense [N, Cout] block per layer)
__global__ void __launch_bounds__(256) demod_kernel(const float* __restrict__ styles, const float* __restrict__ wsq,
                                                    const int64_t* __restrict__ woff, const int* __restrict__ cin,
                                                    const int64_t* __restrict__ soff, const int64_t* __restrict__ ooff,
                                                    const int* __restrict__ cout, float* __restrict__ dcoef, int rows, int N) {
    const int lane = threadIdx.x & 31;
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp_global; r < rows; r += nwarps) {
        const float* w = wsq + woff[r];
        const int c = cin[r];
        for (int n = 0; n < N; ++n) {
            const float* s = styles + soff[r] + (int64_t)n * c;
            float acc = 0.f;
            for (int i = lane; i < c; i += 32) { const float sv = s[i]; acc += sv * sv * __ldg(w + i); }
            acc = warp_sum(acc);
            if (lane == 0) dcoef[ooff[r] + (int64_t)n * cout[r]] = rsqrtf(acc + 1e-8f);
        }
    }
}

// ---------------------------------------------------------------------------------------------- modulate + split
// F16: one fp16 single output in hi (lo unused) instead of the split pair.
template <bool F16>
__global__ void __launch_bounds__(256) modulate_split_kernel(const float* __restrict__ x, int64_t npix, int N, int C,
                                                             const float* __restrict__ style, __nv_bfloat16* __restrict__ hi,
                                                             __nv_bfloat16* __restrict__ lo, int cstride, int coff) {
    const int c4n = C >> 2;
    const int64_t total = (int64_t)N * npix * c4n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % c4n);
        const int64_t pix = i / c4n;
        const int n = (int)(pix / npix);
        float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
        if (style) {
            const float4 s = __ldg(reinterpret_cast<const float4*>(style + (int64_t)n * C) + c4);
            v.x *= s.x; v.y *= s.y; v.z *= s.z; v.w *= s.w;
        }
        const int64_t o = pix * cstride + coff + c4 * 4;
        if constexpr (F16) {
            *reinterpret_cast<uint2*>(hi + o) = make_uint2(pack_half2(v.x, v.y), pack_half2(v.z, v.w));
            continue;
        }
        uint2 h, l;
        split_bf16x2(v.x, v.y, h.x, l.x); split_bf16x2(v.z, v.w, h.y, l.y);
        *reinterpret_cast<uint2*>(hi + o) = h;
        *reinterpret_cast<uint2*>(lo + o) = l;
    }
}

// ---------------------------------------------------------------------------------------------- FIR helpers
// [1,3,3,1]/8 per axis; upfirdn2d's 2-D filter is the outer product / 64 (setup_filter, upfirdn2d.py:101-111).  The up path's gain 4
// is 2 per axis.  constexpr, so that unrolled loops take the taps as immediates.
__device__ constexpr float kFirUp[4] = {0.25f, 0.75f, 0.75f, 0.25f};
__device__ constexpr float kFirDown[4] = {0.125f, 0.375f, 0.375f, 0.125f};

struct EpiParams {
    const float* dcoef; const float* bias; const float* noise; int64_t noise_nstride;
    float gain, slope, clamp;
    N3DSplitOut out[2];
    float* out_f32; int f32_cstride, f32_coff;
};

// float4 arithmetic, one correctly rounded fma / mul per element.
__device__ __forceinline__ float4 f4_fma(float w, const float4& v, const float4& a) {
    return make_float4(__fmaf_rn(w, v.x, a.x), __fmaf_rn(w, v.y, a.y), __fmaf_rn(w, v.z, a.z), __fmaf_rn(w, v.w, a.w));
}
__device__ __forceinline__ float4 f4_fma4(const float4& w, const float4& v, const float4& a) {
    return make_float4(__fmaf_rn(w.x, v.x, a.x), __fmaf_rn(w.y, v.y, a.y), __fmaf_rn(w.z, v.z, a.z), __fmaf_rn(w.w, v.w, a.w));
}
__device__ __forceinline__ float4 f4_mul4(const float4& w, const float4& v) {
    return make_float4(__fmul_rn(w.x, v.x), __fmul_rn(w.y, v.y), __fmul_rn(w.z, v.z), __fmul_rn(w.w, v.w));
}
__device__ __forceinline__ float4 f4_scale(float w, const float4& v) {
    return make_float4(__fmul_rn(w, v.x), __fmul_rn(w, v.y), __fmul_rn(w, v.z), __fmul_rn(w, v.w));
}

// Per-thread epilogue constants of one (image, 4-channel group): demodulation and bias pre-multiplied by the activation gain
// (lrelu(a) * g == lrelu(a * g) for g > 0), the two consumers' styles.
struct EpiVec { float4 dcg, bsg, st[2]; };

__device__ __forceinline__ EpiVec epi_load(const EpiParams& E, int n, int C, int c0) {
    EpiVec V;
    float4 dc = make_float4(1.f, 1.f, 1.f, 1.f), bs = make_float4(0.f, 0.f, 0.f, 0.f);
    if (E.dcoef) dc = __ldg(reinterpret_cast<const float4*>(E.dcoef + (int64_t)n * C + c0));
    if (E.bias) bs = __ldg(reinterpret_cast<const float4*>(E.bias + c0));
    V.dcg = f4_scale(E.gain, dc); V.bsg = f4_scale(E.gain, bs);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        V.st[k] = make_float4(1.f, 1.f, 1.f, 1.f);
        if (E.out[k].hi && E.out[k].style) V.st[k] = __ldg(reinterpret_cast<const float4*>(E.out[k].style + (int64_t)n * C + c0));
    }
    return V;
}

// Output cursors of one thread: element offsets of its current 2x2 block's top-left pixel in the fp32 output and in the two split
// outputs (channel offset included), advanced by two rows per strip step -- no 64-bit multiplies in the loop.
struct EpiCursor { int64_t f32, sp[2]; };

__device__ __forceinline__ EpiCursor epi_cursor(const EpiParams& E, int64_t pix, int c0) {
    EpiCursor P;
    P.f32 = pix * E.f32_cstride + E.f32_coff + c0;
    P.sp[0] = pix * E.out[0].cstride + E.out[0].coff + c0;
    P.sp[1] = pix * E.out[1].cstride + E.out[1].coff + c0;
    return P;
}

// Advances the cursor by two output rows of W2 pixels: the next 2x2 block of a strip.
__device__ __forceinline__ void epi_advance2(EpiCursor& P, const EpiParams& E, int W2) {
    const int64_t rows2 = 2 * (int64_t)W2;
    P.f32 += rows2 * E.f32_cstride;
    P.sp[0] += rows2 * E.out[0].cstride;
    P.sp[1] += rows2 * E.out[1].cstride;
}

// bias_act (lrelu with 0 <= slope <= 1: max(t, slope * t)) + clamp + the fp32 / modulated split-bf16 (or fp16 single) stores of one
// pixel.
// nzg = noise * gain; dpix = pixel offset from the cursor (0, 1, W2, W2 + 1).
__device__ __forceinline__ void epi_store(const EpiParams& E, const EpiVec& V, const EpiCursor& P, const float4& acc, float nzg, int dpix) {
    float4 t = f4_fma4(acc, V.dcg, make_float4(V.bsg.x + nzg, V.bsg.y + nzg, V.bsg.z + nzg, V.bsg.w + nzg));
    const float4 ts = f4_scale(E.slope, t);
    t = make_float4(fmaxf(t.x, ts.x), fmaxf(t.y, ts.y), fmaxf(t.z, ts.z), fmaxf(t.w, ts.w));
    if (E.clamp >= 0.f) {
        const float c = E.clamp;
        t = make_float4(fminf(fmaxf(t.x, -c), c), fminf(fmaxf(t.y, -c), c), fminf(fmaxf(t.z, -c), c), fminf(fmaxf(t.w, -c), c));
    }
    if (E.out_f32) *reinterpret_cast<float4*>(E.out_f32 + P.f32 + dpix * E.f32_cstride) = t;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const N3DSplitOut o = E.out[k];
        if (!o.hi) continue;
        const float4 m = f4_mul4(t, V.st[k]);
        const int64_t off = P.sp[k] + dpix * o.cstride;
        if (o.f16) {
            *reinterpret_cast<uint2*>((__half*)o.hi + off) = make_uint2(pack_half2(m.x, m.y), pack_half2(m.z, m.w));
            continue;
        }
        uint2 h, l;
        split_bf16x2(m.x, m.y, h.x, l.x); split_bf16x2(m.z, m.w, h.y, l.y);
        *reinterpret_cast<uint2*>((__nv_bfloat16*)o.hi + off) = h;
        *reinterpret_cast<uint2*>((__nv_bfloat16*)o.lo + off) = l;
    }
}

// The four FIR kernels share their arithmetic through the helpers below (that is what keeps the register-tiled and the streamed
// forms bit-identical); each kernel keeps only its own work decomposition and data movement.  A thread filters a 2x2 output block
// per strip step from a window of five horizontally filtered input rows h[0..4], two float4 outputs per row.

// One float4 load of a horizontal pass: __ldg from global memory (register-tiled kernels) or a plain shared-memory load (streamed
// kernels, from the row ring).
template <bool GLOBAL>
__device__ __forceinline__ float4 fir_ld(const float4* p) {
    if constexpr (GLOBAL) return __ldg(p);
    else return *p;
}

// Horizontal pass of the up path over one raw row: the outputs that start at raw columns x0-1 and x0, from the five columns
// x0-1 .. x0+3 at p, p + cs, ..., p + 4 cs.  Only the first / last column can fall outside the image (flags vl / vr); a row outside
// the image (in == false) is zero padding and `p` is not read.
template <bool GLOBAL>
__device__ __forceinline__ void fir_up_hrow(const float4* __restrict__ p, bool in, int cs, bool vl, bool vr, float4 (&h)[2]) {
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    h[0] = z; h[1] = z;
    if (!in) return;
    float4 v[5];
    v[0] = vl ? fir_ld<GLOBAL>(p) : z;
#pragma unroll
    for (int c = 1; c < 4; ++c) v[c] = fir_ld<GLOBAL>(p + c * cs);
    v[4] = vr ? fir_ld<GLOBAL>(p + 4 * cs) : z;
#pragma unroll
    for (int b = 0; b < 2; ++b) {
        h[b] = f4_scale(kFirUp[0], v[b]);
#pragma unroll
        for (int fx = 1; fx < 4; ++fx) h[b] = f4_fma(kFirUp[fx], v[b + fx], h[b]);
    }
}

// Vertical pass of the up path over the window h (raw rows y0-1 .. y0+3) and the epilogue of the 2x2 output block at the cursor
// (nzg = noise * gain per output pixel); then the window slides down two rows.
__device__ __forceinline__ void fir_up_vstore(const EpiParams& E, const EpiVec& V, const EpiCursor& P, int W2, const float (&nzg)[2][2],
                                              float4 (&h)[5][2]) {
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            float4 acc = f4_scale(kFirUp[0], h[a][b]);
#pragma unroll
            for (int r = 1; r < 4; ++r) acc = f4_fma(kFirUp[r], h[a + r][b], acc);
            epi_store(E, V, P, acc, nzg[a][b], a * W2 + b);
        }
#pragma unroll
    for (int r = 0; r < 3; ++r) { h[r][0] = h[r + 2][0]; h[r][1] = h[r + 2][1]; }
}

// Horizontal pass of the down path, whose window starts two columns left of x0 (input columns x0-2 .. x0+2, x0 even in [0, W]): the
// first two are outside together (x0 == 0: vl), the next two together (x0 == W: vm), the last one when x0 + 2 >= W (vr).  Rows
// outside the image as in fir_up_hrow.
template <bool GLOBAL>
__device__ __forceinline__ void fir_down_hrow(const float4* __restrict__ p, bool in, int cs, bool vl, bool vm, bool vr, float4 (&h)[2]) {
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    h[0] = z; h[1] = z;
    if (!in) return;
    float4 v[5];
    v[0] = vl ? fir_ld<GLOBAL>(p) : z; v[1] = vl ? fir_ld<GLOBAL>(p + cs) : z;
    v[2] = vm ? fir_ld<GLOBAL>(p + 2 * cs) : z; v[3] = vm ? fir_ld<GLOBAL>(p + 3 * cs) : z;
    v[4] = vr ? fir_ld<GLOBAL>(p + 4 * cs) : z;
    h[0] = f4_scale(kFirDown[0], v[0]); h[1] = f4_scale(kFirDown[0], v[1]);
#pragma unroll
    for (int fx = 1; fx < 4; ++fx) { h[0] = f4_fma(kFirDown[fx], v[fx], h[0]); h[1] = f4_fma(kFirDown[fx], v[fx + 1], h[1]); }
}

// Vertical pass of the down path over the window h (input rows y0-2 .. y0+2): the FIR outputs (y0 + a, x0 + b), zero beyond the
// (H+1)x(W+1) output, stored as split bf16 to parity image 2a + b at element offset o (parity images par_stride apart); then the
// window slides down two rows.
__device__ __forceinline__ void fir_down_vstore(float4 (&h)[5][2], int y0, int x0, int H, int W, int64_t o, int64_t par_stride,
                                                __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            float4 v = f4_scale(kFirDown[0], h[a][b]);
#pragma unroll
            for (int r = 1; r < 4; ++r) v = f4_fma(kFirDown[r], h[a + r][b], v);
            if (y0 + a > H || x0 + b > W) v = make_float4(0.f, 0.f, 0.f, 0.f);     // beyond the (H+1)x(W+1) FIR output: zero pad
            uint2 hh, l;
            split_bf16x2(v.x, v.y, hh.x, l.x); split_bf16x2(v.z, v.w, hh.y, l.y);
            const int64_t off = (int64_t)(a * 2 + b) * par_stride + o;
            *reinterpret_cast<uint2*>(hi + off) = hh;
            *reinterpret_cast<uint2*>(lo + off) = l;
        }
#pragma unroll
    for (int r = 0; r < 3; ++r) { h[r][0] = h[r + 2][0]; h[r][1] = h[r + 2][1]; }
}

// Streamed FIR kernels: kFsConsumers consumer threads and one producer warp per CTA.
constexpr int kFsConsumers = 256, kFsThreads = kFsConsumers + 32;

// Row ring of the streamed FIR kernels in dynamic shared memory: NR stages of row_bytes (one input row segment each), then NR full
// and NR empty mbarriers.  One producer thread fills the stages with 1-D bulk copies; each consumer warp releases a stage once its
// lanes have read it.  Producer and consumers walk the same rows in the same order and skip the same rows outside the image.
struct FirRing {
    uint8_t* smem;
    uint32_t row_bytes, bars;
    int NR, s;              // stage count, current stage
    uint32_t ph;            // parity of the current stage's phase

    __device__ FirRing(uint8_t* smem_, int NR_, uint32_t row_bytes_)
        : smem(smem_), row_bytes(row_bytes_), bars(n3d_tc::smem_u32(smem_) + (uint32_t)NR_ * row_bytes_), NR(NR_), s(0), ph(0) {}
    __device__ uint32_t full_bar(int k) const { return bars + 8u * (uint32_t)k; }
    __device__ uint32_t empty_bar(int k) const { return bars + 8u * (uint32_t)(NR + k); }
    __device__ void advance() { if (++s == NR) { s = 0; ph ^= 1u; } }

    // Called by every thread of the CTA: thread 0 initialises the barriers, then the CTA synchronises.
    __device__ void init() const {
        if (threadIdx.x == 0) {
            for (int k = 0; k < NR; ++k) { n3d_tc::mbar_init(full_bar(k), 1); n3d_tc::mbar_init(empty_bar(k), kFsConsumers / 32); }
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
    }

    // Producer (one thread): rows r0 .. r1 of the NHWC image `img` [rows][cols][C], rows outside [0, rows) skipped (zero padding).  Each
    // stage receives columns c0 .. c1 of one row clipped to the image, a contiguous segment placed so that column c0 + i is always at
    // byte i * C * 4 of the stage.
    __device__ void produce(const float* img, int rows, int cols, int C, int r0, int r1, int c0, int c1) {
        using namespace n3d_tc;
        const int col_lo = max(c0, 0), col_hi = min(c1, cols - 1);
        const uint32_t bytes = (uint32_t)(col_hi - col_lo + 1) * (uint32_t)C * 4u;
        const uint32_t dst = smem_u32(smem) + (uint32_t)(col_lo - c0) * (uint32_t)C * 4u;
        const float* src = img + (int64_t)col_lo * C;
        for (int r = r0; r <= r1; ++r) {
            if (r < 0 || r >= rows) continue;
            mbar_wait_short(empty_bar(s), ph ^ 1u);
            mbar_expect_tx(full_bar(s), bytes);
            bulk_load_1d(dst + (uint32_t)s * row_bytes, src + (int64_t)r * cols * C, bytes, full_bar(s));
            advance();
        }
    }

    // Consumer: waits until the current stage has landed and returns `p` (a location in stage 0) moved to it.
    __device__ const float4* acquire(const float4* p) const {
        n3d_tc::mbar_wait_short(full_bar(s), ph);
        return reinterpret_cast<const float4*>(reinterpret_cast<const uint8_t*>(p) + s * row_bytes);
    }
    // Consumer: every lane of the warp has read the current stage; lane 0 hands it back to the producer.
    __device__ void release(int lane) {
        __syncwarp();
        if (lane == 0) n3d_tc::mbar_arrive(empty_bar(s));
        advance();
    }
};

// thread = (image, strip of S vertically adjacent output row pairs, 2 output columns, 4-channel group).  The 4x4 FIR is separable
// ([1,3,3,1]/8 * 2 per axis).  A 2x2 output block needs 5 raw rows x 4 raw columns; consecutive blocks of the strip share 3 of the
// 5 rows, so the horizontally filtered rows are kept in registers and slid down the strip: 10 float4 loads per 4 outputs instead
// of 25 (the unshared form is bound by L2->L1 traffic, 2.5x the raw tensor).
__global__ void __launch_bounds__(256) fir_up_epilogue_kernel(const float* __restrict__ raw, int N, int H2, int W2, int C, int S, EpiParams E) {
    const int RH = H2 + 1, RW = W2 + 1, c4n = C >> 2, BH = H2 >> 1, BW = W2 / 2, nstrip = (BH + S - 1) / S;
    const int64_t total = (int64_t)N * nstrip * BW * c4n;
    const int64_t rstride = (int64_t)RW * c4n;                  // raw row stride in float4
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % c4n);
        int64_t t = i / c4n;
        const int bx = (int)(t % BW); t /= BW;
        const int st = (int)(t % nstrip);
        const int n = (int)(t / nstrip);
        const int x0 = bx * 2, c0 = c4 * 4;
        const int by_begin = st * S, by_end = min(by_begin + S, BH);
        const bool vl = x0 > 0, vr = x0 + 3 < RW;               // raw columns x0-1 .. x0+3
        // float4 pointer to raw(n, row 0, column x0-1, c0); rows are addressed relative to it
        const float4* col = reinterpret_cast<const float4*>(raw) + ((int64_t)n * RH * RW + (x0 - 1)) * c4n + c4;
        auto hrow = [&](int ry, float4 (&h)[2]) { fir_up_hrow<true>(col + ry * rstride, ry >= 0 && ry < RH, c4n, vl, vr, h); };
        const EpiVec V = epi_load(E, n, C, c0);
        const float* nzp = E.noise ? E.noise + (int64_t)n * E.noise_nstride + x0 : nullptr;
        float4 h[5][2];
#pragma unroll
        for (int r = 0; r < 3; ++r) hrow(2 * by_begin - 1 + r, h[r]);
        EpiCursor P = epi_cursor(E, ((int64_t)n * H2 + 2 * by_begin) * W2 + x0, c0);
        for (int by = by_begin; by < by_end; ++by, epi_advance2(P, E, W2)) {
            const int y0 = by * 2;
            hrow(y0 + 2, h[3]);
            hrow(y0 + 3, h[4]);
            float nzg[2][2];
#pragma unroll
            for (int a = 0; a < 2; ++a)
#pragma unroll
                for (int b = 0; b < 2; ++b) nzg[a][b] = nzp ? __fmul_rn(E.gain, __ldg(nzp + (int64_t)(y0 + a) * W2 + b)) : 0.f;   // explicit: no FMA contraction into the bias add
            fir_up_vstore(E, V, P, W2, nzg, h);
        }
    }
}

// ---------------------------------------------------------------------------------------------- streamed FIR-up epilogue
// Same arithmetic as fir_up_epilogue_kernel (bit-identical results), different data movement.  The register-tiled kernel above is
// bound by load latency at 16 warps/SM: every strip step waits for its own ten 16-byte loads.  Here a CTA owns a (TR output rows)
// x (TC output columns) x (all C channels) tile of one image and a producer thread streams the raw rows it needs -- each a
// CONTIGUOUS (TC + 3) * C * 4-byte segment of the NHWC tensor -- through the row ring; the eight consumer warps read the five
// columns of their 2-column output block from shared memory.  Loads are in flight NR rows ahead of the arithmetic and cost no
// registers.  thread = (column pair, 4-channel group): (TC / 2) * (C / 4) == 256.
__global__ void __launch_bounds__(kFsThreads, 2) fir_up_stream_kernel(const float* __restrict__ raw, int N, int H2, int W2, int C, int TC, int TR, int NR,
                                                                       EpiParams E) {
    extern __shared__ __align__(128) uint8_t fs_smem[];
    const int RH = H2 + 1, RW = W2 + 1, c4n = C >> 2;
    FirRing ring(fs_smem, NR, (uint32_t)(TC + 3) * (uint32_t)C * 4u);
    const int tiles_x = W2 / TC, tiles_y = H2 / TR;
    const int bx = blockIdx.x % tiles_x, by = (blockIdx.x / tiles_x) % tiles_y, n = blockIdx.x / (tiles_x * tiles_y);
    const int X0 = bx * TC, Y0 = by * TR;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    ring.init();

    if (warp == kFsConsumers / 32) {                            // producer: raw rows Y0-1 .. Y0+TR+1, columns X0-1 .. X0+TC+1
        if (lane == 0) ring.produce(raw + (int64_t)n * RH * RW * C, RH, RW, C, Y0 - 1, Y0 + TR + 1, X0 - 1, X0 + TC + 1);
        return;
    }

    // ========================================================= consumers
    const int c4 = threadIdx.x % c4n, j = threadIdx.x / c4n;
    const int x0 = X0 + 2 * j, c0 = c4 * 4;
    const bool vl = x0 > 0, vr = x0 + 3 < RW;                   // raw columns x0-1 .. x0+3
    const float4* base = reinterpret_cast<const float4*>(fs_smem) + (2 * j) * c4n + c4;      // raw column x0-1 in stage 0
    auto hrow = [&](int ry, float4 (&h)[2]) {                  // one call: written as in fir_down_stream_kernel, this kernel spills
        const bool in = ry >= 0 && ry < RH;
        fir_up_hrow<false>(in ? ring.acquire(base) : nullptr, in, c4n, vl, vr, h);
        if (in) ring.release(lane);
    };
    const EpiVec V = epi_load(E, n, C, c0);
    const float* nzp = E.noise ? E.noise + (int64_t)n * E.noise_nstride + x0 : nullptr;
    float4 h[5][2];
#pragma unroll
    for (int r = 0; r < 3; ++r) hrow(Y0 - 1 + r, h[r]);
    EpiCursor P = epi_cursor(E, ((int64_t)n * H2 + Y0) * W2 + x0, c0);
    // the noise of a 2x2 block is fetched one strip step ahead, so that its global-load latency does not sit between the FIR and the
    // stores
    float nzn[2][2];
    auto load_noise = [&](int y0) {
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 2; ++b) nzn[a][b] = nzp ? __ldg(nzp + (int64_t)(y0 + a) * W2 + b) : 0.f;
    };
    load_noise(Y0);
    for (int y0 = Y0; y0 < Y0 + TR; y0 += 2, epi_advance2(P, E, W2)) {
        float nzg[2][2];
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 2; ++b) nzg[a][b] = __fmul_rn(E.gain, nzn[a][b]);     // same rounding as the register-tiled kernel
        if (y0 + 2 < Y0 + TR) load_noise(y0 + 2);
        hrow(y0 + 2, h[3]);
        hrow(y0 + 3, h[4]);
        fir_up_vstore(E, V, P, W2, nzg, h);
    }
}

// Second pass of a split-K convolution: sum the S raw partial tensors in a fixed order, then the usual epilogue.
// thread = (pixel, 4-channel group).
__global__ void __launch_bounds__(256) splitk_epilogue_kernel(const float* __restrict__ part, int S, int64_t stride, int N, int H, int W, int C, EpiParams E) {
    const int c4n = C >> 2;
    const int64_t total = (int64_t)N * H * W * c4n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % c4n);
        const int64_t pix = i / c4n;
        const int n = (int)(pix / ((int64_t)H * W));
        const int64_t yx = pix - (int64_t)n * H * W;
        float4 acc = __ldg(reinterpret_cast<const float4*>(part) + i);
        for (int s = 1; s < S; ++s) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(part + (int64_t)s * stride) + i);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        const EpiVec V = epi_load(E, n, C, c4 * 4);
        const EpiCursor P = epi_cursor(E, pix, c4 * 4);
        const float nzg = E.noise ? __fmul_rn(E.gain, __ldg(E.noise + (int64_t)n * E.noise_nstride + yx)) : 0.f;
        epi_store(E, V, P, acc, nzg, 0);
    }
}

// FIR (pad 2,2,2,2) -> [(H+1),(W+1)] -> parity-split bf16 hi/lo, layout [4 parities][N][SH][SW][C].
// thread = (image, strip of S sub-pixel rows, sub-pixel column sx, 4-channel group) -> per sub-pixel the 2x2 block of FIR outputs
// (2sy+a, 2sx+b), one per parity image; same register-resident sliding window over the horizontally filtered rows as above.
__global__ void __launch_bounds__(256) fir_down_split_kernel(const float* __restrict__ x, int N, int H, int W, int C, int S,
                                                             __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    const int SH = (H + 2) / 2, SW = (W + 2) / 2, c4n = C >> 2, nstrip = (SH + S - 1) / S;
    const int64_t total = (int64_t)N * nstrip * SW * c4n;
    const int64_t par_stride = (int64_t)N * SH * SW * C;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % c4n);
        int64_t t = i / c4n;
        const int sx = (int)(t % SW); t /= SW;
        const int st = (int)(t % nstrip);
        const int n = (int)(t / nstrip);
        const int x0 = sx * 2;                               // FIR output (y, x) reads input rows y-2 .. y+1, columns x-2 .. x+1
        const int sy_begin = st * S, sy_end = min(sy_begin + S, SH);
        const bool vl = x0 >= 2, vm = x0 < W, vr = x0 + 2 < W;
        const float4* col = reinterpret_cast<const float4*>(x) + ((int64_t)n * H * W + (x0 - 2)) * c4n + c4;
        const int64_t rstride = (int64_t)W * c4n;
        auto hrow = [&](int iy, float4 (&h)[2]) { fir_down_hrow<true>(col + iy * rstride, iy >= 0 && iy < H, c4n, vl, vm, vr, h); };
        float4 h[5][2];
#pragma unroll
        for (int r = 0; r < 3; ++r) hrow(2 * sy_begin - 2 + r, h[r]);
        for (int sy = sy_begin; sy < sy_end; ++sy) {
            const int y0 = sy * 2;
            hrow(y0 + 1, h[3]);
            hrow(y0 + 2, h[4]);
            fir_down_vstore(h, y0, x0, H, W, (((int64_t)n * SH + sy) * SW + sx) * C + c4 * 4, par_stride, hi, lo);
        }
    }
}

// Streamed form of fir_down_split_kernel (same arithmetic, bit-identical), built like fir_up_stream_kernel: a CTA owns TS sub-pixel rows x
// TSC sub-pixel columns x all channels of one image ((TSC) * (C / 4) == 256 consumer threads) and a producer thread streams the
// 2 TS + 3 input rows -- contiguous (2 TSC + 3) * C * 4-byte segments -- through the shared-memory ring with 1-D bulk copies.
__global__ void __launch_bounds__(kFsThreads, 2) fir_down_stream_kernel(const float* __restrict__ x, int N, int H, int W, int C, int TSC, int TS, int NR,
                                                                         __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    extern __shared__ __align__(128) uint8_t fs_smem[];
    const int SH = (H + 2) / 2, SW = (W + 2) / 2, c4n = C >> 2;
    FirRing ring(fs_smem, NR, (uint32_t)(2 * TSC + 3) * (uint32_t)C * 4u);
    const int tiles_x = (SW + TSC - 1) / TSC, tiles_y = (SH + TS - 1) / TS;
    const int bx = blockIdx.x % tiles_x, by = (blockIdx.x / tiles_x) % tiles_y, n = blockIdx.x / (tiles_x * tiles_y);
    const int SX0 = bx * TSC, SY0 = by * TS, rows_here = min(TS, SH - SY0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    ring.init();
    const int iy_first = 2 * SY0 - 2, iy_last = 2 * (SY0 + rows_here - 1) + 2;

    if (warp == kFsConsumers / 32) {                            // producer: input columns 2 SX0 - 2 .. 2 SX0 + 2 TSC
        if (lane == 0) ring.produce(x + (int64_t)n * H * W * C, H, W, C, iy_first, iy_last, 2 * SX0 - 2, 2 * SX0 + 2 * TSC);
        return;
    }

    const int c4 = threadIdx.x % c4n, j = threadIdx.x / c4n;
    const int sx = SX0 + j, x0 = 2 * sx;
    const bool active = sx < SW;                                // the last column tile is ragged (SW = W / 2 + 1)
    const bool vl = active && x0 >= 2, vm = active && x0 < W, vr = active && x0 + 2 < W;
    const float4* base = reinterpret_cast<const float4*>(fs_smem) + (2 * j) * c4n + c4;      // input column x0 - 2 in stage 0
    auto hrow = [&](int iy, float4 (&h)[2]) {                  // two calls: fewer instructions per row than fir_up_stream_kernel's form
        if (iy < 0 || iy >= H) return fir_down_hrow<false>(nullptr, false, c4n, vl, vm, vr, h);
        fir_down_hrow<false>(ring.acquire(base), true, c4n, vl, vm, vr, h);
        ring.release(lane);
    };
    const int64_t par_stride = (int64_t)N * SH * SW * C;
    float4 h[5][2];                                             // all zero in an inactive thread: it needs no slide
#pragma unroll
    for (int r = 0; r < 3; ++r) hrow(iy_first + r, h[r]);
    for (int sy = SY0; sy < SY0 + rows_here; ++sy) {
        const int y0 = sy * 2;
        hrow(y0 + 1, h[3]);
        hrow(y0 + 2, h[4]);
        if (active) fir_down_vstore(h, y0, x0, H, W, (((int64_t)n * SH + sy) * SW + sx) * C + c4 * 4, par_stride, hi, lo);
    }
}

// upsample2d: zero-insert x2, pad (2,1), 4x4 FIR * 4.  Polyphase form: out[2i] = .25 x[i-1] + .75 x[i], out[2i+1] = .75 x[i] + .25 x[i+1]
// per axis.  thread = (input pixel (i,j), VEC channels) -> the 2x2 output block from the 3x3 input neighbourhood.
template <int VEC>
__global__ void __launch_bounds__(256) upsample2d_kernel(const float* __restrict__ x, int N, int H, int W, int C, float* __restrict__ y, int nchw) {
    const int OH = 2 * H, OW = 2 * W, cvn = C / VEC;
    const int64_t total = (int64_t)N * H * W * cvn;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int cv = (int)(idx % cvn);
        int64_t t = idx / cvn;
        const int j = (int)(t % W); t /= W;
        const int i = (int)(t % H);
        const int n = (int)(t / H);
        float v[3][3][VEC];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) {
                const int yy = i - 1 + a, xx = j - 1 + b;
                const bool ok = yy >= 0 && yy < H && xx >= 0 && xx < W;
                const float* src = x + (((int64_t)n * H + (ok ? yy : 0)) * W + (ok ? xx : 0)) * C + cv * VEC;
                if (VEC == 4) {
                    const float4 q = ok ? __ldg(reinterpret_cast<const float4*>(src)) : make_float4(0.f, 0.f, 0.f, 0.f);
                    v[a][b][0] = q.x; v[a][b][1 % VEC] = q.y; v[a][b][2 % VEC] = q.z; v[a][b][3 % VEC] = q.w;
                } else {
                    v[a][b][0] = ok ? __ldg(src) : 0.f;
                }
            }
        const float wa[2][3] = {{0.25f, 0.75f, 0.f}, {0.f, 0.75f, 0.25f}};
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 2; ++b) {
                float o[VEC];
#pragma unroll
                for (int e = 0; e < VEC; ++e) {
                    float acc = 0.f;
#pragma unroll
                    for (int p = 0; p < 3; ++p)
#pragma unroll
                        for (int q = 0; q < 3; ++q) acc += (wa[a][p] * wa[b][q]) * v[p][q][e];
                    o[e] = acc;
                }
                const int oy = 2 * i + a, ox = 2 * j + b;
                if (nchw) {
#pragma unroll
                    for (int e = 0; e < VEC; ++e) y[(((int64_t)n * C + cv * VEC + e) * OH + oy) * OW + ox] = o[e];
                } else {
                    float* dst = y + (((int64_t)n * OH + oy) * OW + ox) * C + cv * VEC;
                    if (VEC == 4) *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1 % VEC], o[2 % VEC], o[3 % VEC]);
                    else dst[0] = o[0];
                }
            }
    }
}

// downsample2d: pad (1,1), 4x4 FIR, keep every 2nd pixel
__global__ void __launch_bounds__(256) downsample2d_kernel(const float* __restrict__ x, int N, int H, int W, int C, float* __restrict__ y) {
    const int OH = H / 2, OW = W / 2;
    const int64_t total = (int64_t)N * OH * OW * C;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        int64_t t = i / C;
        const int ox = (int)(t % OW); t /= OW;
        const int oy = (int)(t % OH);
        const int n = (int)(t / OH);
        float acc = 0.f;
#pragma unroll
        for (int fy = 0; fy < 4; ++fy) {
            const int iy = oy * 2 + fy - 1;
            if (iy < 0 || iy >= H) continue;
#pragma unroll
            for (int fx = 0; fx < 4; ++fx) {
                const int ix = ox * 2 + fx - 1;
                if (ix < 0 || ix >= W) continue;
                acc += (kFirDown[fy] * kFirDown[fx]) * __ldg(x + (((int64_t)n * H + iy) * W + ix) * C + c);
            }
        }
        y[i] = acc;
    }
}
}  // namespace

extern "C" int n3d_styles(const float* ws, int N, int num_ws, int wdim, const float* affine_w, const float* affine_b,
                          const int32_t* row_widx, const float* row_scale, const int64_t* row_ooff, const int32_t* row_cin,
                          float* styles, int rows, void* stream) {
    N3D_CHECK_ARG(ws && affine_w && affine_b && row_widx && row_scale && row_ooff && row_cin && styles, "n3d_styles: null pointer");
    N3D_CHECK_ARG(wdim % 4 == 0 && rows > 0 && N > 0, "n3d_styles: bad sizes");
    N3D_CHECK_ARG((((uintptr_t)ws | (uintptr_t)affine_w) & 15) == 0, "n3d_styles: ws and affine_w must be 16-byte aligned");   // float4 loads
    styles_kernel<<<n3d_grid((int64_t)rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(ws, N, num_ws, wdim, affine_w, affine_b, row_widx,
                                                                                      row_scale, row_ooff, row_cin, styles, rows);
    N3D_CHECK_LAUNCH("n3d_styles");
    return N3D_OK;
}

extern "C" int n3d_demod(const float* styles, const float* wsq, const int64_t* row_woff, const int32_t* row_cin,
                         const int64_t* row_soff, const int64_t* row_ooff, const int32_t* row_cout, float* dcoef, int rows, int N,
                         void* stream) {
    N3D_CHECK_ARG(styles && wsq && row_woff && row_cin && row_soff && row_ooff && row_cout && dcoef, "n3d_demod: null pointer");
    demod_kernel<<<n3d_grid((int64_t)rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(styles, wsq, row_woff, row_cin, row_soff, row_ooff,
                                                                                     row_cout, dcoef, rows, N);
    N3D_CHECK_LAUNCH("n3d_demod");
    return N3D_OK;
}

// Rows per thread strip of the FIR kernels: 16 (3 re-read halo rows per strip) for launches with >= 1024 threads per SM, halved
// down to 4 for smaller ones: longer strips re-read fewer halo rows, shorter ones keep small launches filling the SMs.
static int fir_strip_rows(int num_sms, int64_t threads_per_row, int rows) {
    int S = 16;
    while (S > 4 && threads_per_row * n3d_div_up(rows, S) < (int64_t)num_sms * 1024) S >>= 1;
    return min(S, rows);
}

// N3D_FIR_STREAM=0: the register-tiled FIR kernels everywhere (the reference of the streamed ones in the bit-identity tests).  Read
// at call time so that one process can run both forms.
static bool fir_stream_enabled() {
    const char* e = getenv("N3D_FIR_STREAM");
    return !e || atoi(e) != 0;
}

// Epilogue descriptor of n3d_fir_up_epilogue and n3d_splitk_epilogue, with the checks both need of it.  epi_load reads dcoef,
// bias and the styles as float4, epi_store writes float4 / uint2: strides, offsets and base pointers must all keep that alignment.
static int make_epi(EpiParams* E, const char* who, const float* dcoef, const float* bias, const float* noise, int64_t noise_nstride,
                    float gain, float slope, float clamp, const N3DSplitOut out[2], float* out_f32, int f32_cstride, int f32_coff) {
    N3D_CHECK_ARG(gain > 0.f && slope >= 0.f && slope <= 1.f, "%s: needs gain > 0 and 0 <= slope <= 1 (lrelu / linear)", who);
    for (int k = 0; k < 2; ++k) {
        N3D_CHECK_ARG(!out[k].hi || (out[k].cstride % 4 == 0 && out[k].coff % 4 == 0), "%s: unaligned split output", who);
        N3D_CHECK_ARG(!out[k].hi || (((uintptr_t)out[k].hi | (uintptr_t)out[k].lo | (uintptr_t)out[k].style) & 15) == 0,
                      "%s: split output %d (hi / lo / style) must be 16-byte aligned", who, k);
        N3D_CHECK_ARG(!out[k].hi || out[k].f16 == 1 || (out[k].f16 == 0 && out[k].lo), "%s: output %d: f16 must be 0 (split bf16, hi and lo) or 1 "
                      "(fp16 single)", who, k);
    }
    N3D_CHECK_ARG(!out_f32 || (f32_cstride % 4 == 0 && f32_coff % 4 == 0), "%s: unaligned fp32 output", who);
    N3D_CHECK_ARG(((uintptr_t)out_f32 & 15) == 0, "%s: out_f32 must be 16-byte aligned", who);
    N3D_CHECK_ARG((((uintptr_t)dcoef | (uintptr_t)bias) & 15) == 0, "%s: dcoef and bias must be 16-byte aligned", who);
    *E = EpiParams{dcoef, bias, noise, noise_nstride, gain, slope, clamp, {out[0], out[1]}, out_f32, f32_cstride, f32_coff};
    return N3D_OK;
}

extern "C" int n3d_modulate_split(const float* x, int64_t npix_per_img, int N, int C, const float* style, void* hi, void* lo,
                                  int out_cstride, int out_coff, void* stream) {
    N3D_CHECK_ARG(x && hi && lo, "n3d_modulate_split: null pointer");
    N3D_CHECK_ARG(C % 4 == 0 && out_cstride % 4 == 0 && out_coff % 4 == 0, "n3d_modulate_split: channels must be multiples of 4");
    N3D_CHECK_ARG((((uintptr_t)x | (uintptr_t)style) & 15) == 0, "n3d_modulate_split: x and style must be 16-byte aligned");   // float4 loads
    N3D_CHECK_ARG((((uintptr_t)hi | (uintptr_t)lo) & 7) == 0, "n3d_modulate_split: hi and lo must be 8-byte aligned");          // uint2 stores
    const int64_t total = (int64_t)N * npix_per_img * (C / 4);
    modulate_split_kernel<false><<<n3d_grid(total, 256, 16), 256, 0, (cudaStream_t)stream>>>(x, npix_per_img, N, C, style, (__nv_bfloat16*)hi,
                                                                                            (__nv_bfloat16*)lo, out_cstride, out_coff);
    N3D_CHECK_LAUNCH("n3d_modulate_split");
    return N3D_OK;
}

extern "C" int n3d_modulate_f16(const float* x, int64_t npix_per_img, int N, int C, const float* style, void* out, int out_cstride,
                                int out_coff, void* stream) {
    N3D_CHECK_ARG(x && out, "n3d_modulate_f16: null pointer");
    N3D_CHECK_ARG(C % 4 == 0 && out_cstride % 4 == 0 && out_coff % 4 == 0, "n3d_modulate_f16: channels must be multiples of 4");
    N3D_CHECK_ARG((((uintptr_t)x | (uintptr_t)style) & 15) == 0, "n3d_modulate_f16: x and style must be 16-byte aligned");     // float4 loads
    N3D_CHECK_ARG(((uintptr_t)out & 7) == 0, "n3d_modulate_f16: out must be 8-byte aligned");                                   // uint2 stores
    const int64_t total = (int64_t)N * npix_per_img * (C / 4);
    modulate_split_kernel<true><<<n3d_grid(total, 256, 16), 256, 0, (cudaStream_t)stream>>>(x, npix_per_img, N, C, style, (__nv_bfloat16*)out,
                                                                                           nullptr, out_cstride, out_coff);
    N3D_CHECK_LAUNCH("n3d_modulate_f16");
    return N3D_OK;
}

extern "C" int n3d_fir_up_epilogue(const float* raw, int N, int H2, int W2, int C, const float* dcoef, const float* bias,
                                   const float* noise, int64_t noise_nstride, float gain, float slope, float clamp,
                                   const N3DSplitOut out[2], float* out_f32, int f32_cstride, int f32_coff, void* stream) {
    N3D_CHECK_ARG(raw && out, "n3d_fir_up_epilogue: null pointer");
    N3D_CHECK_ARG(((uintptr_t)raw & 15) == 0, "n3d_fir_up_epilogue: raw must be 16-byte aligned");     // float4 loads (both kernels)
    N3D_CHECK_ARG(C % 4 == 0, "n3d_fir_up_epilogue: C must be a multiple of 4");
    N3D_CHECK_ARG(H2 % 2 == 0 && W2 % 2 == 0, "n3d_fir_up_epilogue: output size must be even");
    EpiParams E;
    if (int rc = make_epi(&E, "n3d_fir_up_epilogue", dcoef, bias, noise, noise_nstride, gain, slope, clamp, out, out_f32, f32_cstride, f32_coff))
        return rc;
    const N3DDeviceState* D = n3d_device_state();
    if (!D) return N3D_ERR_CUDA;
    const int sms = D->num_sms;
    // streamed variant (fir_up_stream_kernel) for the large layers: (TC / 2) * (C / 4) == 256 consumer threads, >= one CTA per SM.
    // Rows per tile: the candidate with the best (fill of the last wave of 2 CTAs per SM) x (1 - vertical halo).  The tiling does not
    // change the arithmetic (results are bit-identical for every TR).
    const int TC = (C >= 64 && C <= 512 && (2048 % C) == 0) ? 2048 / C : 0;
    int TR = 0;
    if (TC >= 4 && W2 % TC == 0) {
        double best = 0.0;
        for (int tr = 32; tr <= 128; tr *= 2) {
            if (H2 % tr) continue;
            const int64_t ctas = (int64_t)N * (W2 / TC) * (H2 / tr);
            if (ctas < sms) continue;
            const double eff = (double)ctas / (double)(n3d_div_up(ctas, 2 * sms) * 2 * sms) * tr / (tr + 3);
            if (eff > best) { best = eff; TR = tr; }
        }
    }
    if (TR > 0 && fir_stream_enabled()) {
        const int row_bytes = (TC + 3) * C * 4;
        const int NR = min(4, (100 * 1024) / row_bytes);        // ring depth: 4 stages
        const int smem = NR * row_bytes + 16 * NR;
        if (int rc = n3d_smem_optin((const void*)fir_up_stream_kernel, 112 * 1024, "n3d_fir_up_epilogue")) return rc;
        fir_up_stream_kernel<<<N * (W2 / TC) * (H2 / TR), kFsThreads, smem, (cudaStream_t)stream>>>(raw, N, H2, W2, C, TC, TR, NR, E);
        N3D_CHECK_LAUNCH("n3d_fir_up_epilogue");
        return N3D_OK;
    }
    const int S = fir_strip_rows(sms, (int64_t)N * (W2 / 2) * (C / 4), H2 / 2);
    const int64_t total = (int64_t)N * n3d_div_up(H2 / 2, S) * (W2 / 2) * (C / 4);
    // 2 output columns per thread: the two columns share each input row's loads
    fir_up_epilogue_kernel<<<n3d_grid(total, 256, 16), 256, 0, (cudaStream_t)stream>>>(raw, N, H2, W2, C, S, E);
    N3D_CHECK_LAUNCH("n3d_fir_up_epilogue");
    return N3D_OK;
}

extern "C" int n3d_splitk_epilogue(const float* partial, int S, int64_t split_stride, int N, int H, int W, int C, const float* dcoef,
                                   const float* bias, const float* noise, int64_t noise_nstride, float gain, float slope, float clamp,
                                   const N3DSplitOut out[2], float* out_f32, int f32_cstride, int f32_coff, void* stream) {
    N3D_CHECK_ARG(partial && out && S >= 1 && N > 0 && H > 0 && W > 0, "n3d_splitk_epilogue: bad args");
    N3D_CHECK_ARG(C % 4 == 0 && split_stride % 4 == 0 && ((uintptr_t)partial & 15) == 0, "n3d_splitk_epilogue: C and the split stride must be multiples of 4");
    EpiParams E;
    if (int rc = make_epi(&E, "n3d_splitk_epilogue", dcoef, bias, noise, noise_nstride, gain, slope, clamp, out, out_f32, f32_cstride, f32_coff))
        return rc;
    const int64_t total = (int64_t)N * H * W * (C / 4);
    splitk_epilogue_kernel<<<n3d_grid(total, 256, 16), 256, 0, (cudaStream_t)stream>>>(partial, S, split_stride, N, H, W, C, E);
    N3D_CHECK_LAUNCH("n3d_splitk_epilogue");
    return N3D_OK;
}

extern "C" int n3d_fir_down_split(const float* x, int N, int H, int W, int C, void* hi, void* lo, void* stream) {
    N3D_CHECK_ARG(x && hi && lo, "n3d_fir_down_split: null pointer");
    N3D_CHECK_ARG(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, "n3d_fir_down_split: C %% 4 and even H, W required");
    N3D_CHECK_ARG(((uintptr_t)x & 15) == 0, "n3d_fir_down_split: x must be 16-byte aligned");       // float4 loads / bulk copies (both kernels)
    N3D_CHECK_ARG((((uintptr_t)hi | (uintptr_t)lo) & 7) == 0, "n3d_fir_down_split: hi and lo must be 8-byte aligned");     // uint2 stores
    const N3DDeviceState* D = n3d_device_state();
    if (!D) return N3D_ERR_CUDA;
    const int sms = D->num_sms;
    // streamed variant for the large layers (see fir_down_stream_kernel)
    const int c4n = C / 4, SH = (H + 2) / 2, SW = (W + 2) / 2;
    const int TSC = (c4n >= 8 && c4n <= 128 && 256 % c4n == 0) ? 256 / c4n : 0;
    int TS = 0;
    for (int ts = 32; ts >= 16 && TSC; ts >>= 1)
        if ((int64_t)N * n3d_div_up(SW, TSC) * n3d_div_up(SH, ts) >= sms) { TS = ts; break; }
    if (TS > 0 && fir_stream_enabled()) {
        const int row_bytes = (2 * TSC + 3) * C * 4, NR = 4;
        const int smem = NR * row_bytes + 16 * NR;
        if (int rc = n3d_smem_optin((const void*)fir_down_stream_kernel, 112 * 1024, "n3d_fir_down_split")) return rc;
        fir_down_stream_kernel<<<N * n3d_div_up(SW, TSC) * n3d_div_up(SH, TS), kFsThreads, smem, (cudaStream_t)stream>>>(
            x, N, H, W, C, TSC, TS, NR, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
        N3D_CHECK_LAUNCH("n3d_fir_down_split");
        return N3D_OK;
    }
    const int S = fir_strip_rows(sms, (int64_t)N * SW * c4n, SH);
    const int64_t total = (int64_t)N * n3d_div_up(SH, S) * SW * c4n;
    fir_down_split_kernel<<<n3d_grid(total, 256, 16), 256, 0, (cudaStream_t)stream>>>(x, N, H, W, C, S, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
    N3D_CHECK_LAUNCH("n3d_fir_down_split");
    return N3D_OK;
}

extern "C" int n3d_upsample2d_nhwc(const float* x, int N, int H, int W, int C, float* y, int y_nchw, void* stream) {
    N3D_CHECK_ARG(x && y, "n3d_upsample2d_nhwc: null pointer");
    // float4 loads of x and (NHWC) float4 stores of y where the channels and both pointers allow them, else one channel per thread
    if (C % 4 == 0 && ((uintptr_t)x & 15) == 0 && (y_nchw || ((uintptr_t)y & 15) == 0))
        upsample2d_kernel<4><<<n3d_grid((int64_t)N * H * W * (C / 4), 256, 16), 256, 0, (cudaStream_t)stream>>>(x, N, H, W, C, y, y_nchw);
    else
        upsample2d_kernel<1><<<n3d_grid((int64_t)N * H * W * C, 256, 16), 256, 0, (cudaStream_t)stream>>>(x, N, H, W, C, y, y_nchw);
    N3D_CHECK_LAUNCH("n3d_upsample2d_nhwc");
    return N3D_OK;
}

extern "C" int n3d_downsample2d_nhwc(const float* x, int N, int H, int W, int C, float* y, void* stream) {
    N3D_CHECK_ARG(x && y && H % 2 == 0 && W % 2 == 0, "n3d_downsample2d_nhwc: bad args");
    downsample2d_kernel<<<n3d_grid((int64_t)N * (H / 2) * (W / 2) * C, 256, 16), 256, 0, (cudaStream_t)stream>>>(x, N, H, W, C, y);
    N3D_CHECK_LAUNCH("n3d_downsample2d_nhwc");
    return N3D_OK;
}
