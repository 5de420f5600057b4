// Weight gradient of the implicit-GEMM convolutions on Hopper warpgroup tensor cores (wgmma, sm_90a): the backward pass of
// torch_utils.ops.conv2d_resample (next3d_b200/torch_utils/ops/conv2d_resample.py).
//
//   dW[g][t][m][n] = sum_{k < K} A[a_row[t] + g*M + m][k + a_off[t]] * B[b_row[t] + g*N + n][k + b_off[t]]
//
// A (the output gradient) and B (the layer input) are channel-major: one row per channel, one column per position of a padded
// (and for stride-2 taps parity-split) position grid that n3d_wgrad_operand lays out from an NCHW tensor.  A tap is then a constant
// column offset, and reads outside a row's columns are zero-filled by TMA, which is the convolution padding.  A TMA box must start
// on a 16-byte boundary of the row, so column offsets are multiples of 8: the grid rows are padded to a multiple of 8 positions,
// and a horizontal tap shift is a copy of the operand shifted by that many columns, selected by the tap's row offset.  Both operands are
// K-major (positions contiguous), so the shared-memory tiles are the SWIZZLE_128B layout conv_gemm_kernel feeds wgmma.
//   Tile: M = 128 output channels (two m64 wgmmas), N = block_n input channels (32, 64 or 128), K = 64 positions per stage.
//   Precision: the forward's bf16x3 (hi*hi + hi*lo + lo*hi, fp32 accumulate in registers).
//   Grid: x = (m-tile, n-tile, K slice), y = tap, z = group.  K slice s of every tile writes its fp32 partial sums to its own
//   slab; wgrad_reduce_kernel adds the slabs in slice order.  No atomics: the result is the same bit for bit on every run.
//   Warp roles (160 threads): warps 0-3 = one consumer warpgroup (wgmma, then the partial-sum stores), warp 4 = TMA producer (one lane).
#include <cstring>
#include "common.cuh"
#include <cuda.h>
#include "tc_ptx.cuh"

namespace {
using namespace n3d_tc;

constexpr int kBM = 128, kBK = 64;
constexpr int kThreads = 160;
constexpr int kABytes = kBM * kBK * 2;                // one bf16 A tile (hi or lo)
constexpr int kRingBytes = 200 * 1024;
constexpr int kMaxStages = 6;

struct WParams {
    CUtensorMap tmA[2], tmB[2];                        // hi, lo
    int G, M, N, T, splits, stages, stage_bytes, n_tiles;
    int ksteps;                                        // K / 64
    int a_off[9], b_off[9], a_row[9], b_row[9];
    float* out; int64_t slice_stride;                  // K slice s writes out + s * slice_stride
};

template <int BN>
__global__ void __launch_bounds__(kThreads, 1) conv_wgrad_kernel(const __grid_constant__ WParams P) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_base = smem_base + (uint32_t)P.stages * (uint32_t)P.stage_bytes;
    auto full_bar = [&](int s) { return bar_base + 8u * (uint32_t)s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (uint32_t)(P.stages + s); };
    constexpr uint32_t kBBytes = BN * kBK * 2;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int split = blockIdx.x % P.splits, tile = blockIdx.x / P.splits;
    const int nt = tile % P.n_tiles, mt = tile / P.n_tiles;
    const int t = blockIdx.y, g = blockIdx.z;
    const int per = (P.ksteps + P.splits - 1) / P.splits;
    const int kb = min(P.ksteps, split * per), ke = min(P.ksteps, kb + per);

    if (warp == 4 && lane == 0) {
        for (int i = 0; i < 2; ++i) { tma_prefetch_desc(&P.tmA[i]); tma_prefetch_desc(&P.tmB[i]); }
        for (int s = 0; s < P.stages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 4) {
        // ===================================================== TMA producer
        if (lane == 0) {
            int s = 0; uint32_t ph = 0;
            const int arow = P.a_row[t] + g * P.M + mt * kBM, brow = P.b_row[t] + g * P.N + nt * BN;
            const int aoff = P.a_off[t], boff = P.b_off[t];
            for (int ks = kb; ks < ke; ++ks) {
                mbar_wait(empty_bar(s), ph ^ 1u, nullptr, 1);
                const uint32_t sa = smem_base + (uint32_t)s * (uint32_t)P.stage_bytes, fb = full_bar(s);
                mbar_expect_tx(fb, 2u * (kABytes + kBBytes));
                const int k = ks * kBK;
                tma_load_2d(sa, &P.tmA[0], fb, k + aoff, arow);
                tma_load_2d(sa + kABytes, &P.tmA[1], fb, k + aoff, arow);
                tma_load_2d(sa + 2 * kABytes, &P.tmB[0], fb, k + boff, brow);
                tma_load_2d(sa + 2 * kABytes + kBBytes, &P.tmB[1], fb, k + boff, brow);
                if (++s == P.stages) { s = 0; ph ^= 1u; }
            }
        }
        return;
    }

    // ===================================================== consumer warpgroup: conv_gemm_kernel's stage, so the same summation order.
    // Every stage adds to zeroed accumulators (not the FIRST form, which could leave -0 for an all-zero sum).
    float acc0[BN / 2], acc1[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    int s = 0, prev = -1; uint32_t ph = 0;
    for (int ks = kb; ks < ke; ++ks) {
        mbar_wait(full_bar(s), ph, nullptr, 3);
        const uint32_t sa = smem_base + (uint32_t)s * (uint32_t)P.stage_bytes;
        stage_mma<BN, kBK, 3, false>(acc0, acc1, sa, sa + kABytes, sa + 2 * kABytes, sa + 2 * kABytes + kBBytes);
        wgmma_wait<1>();                                 // the previous stage's wgmmas have retired: release it
        __syncwarp();
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        prev = s;
        if (++s == P.stages) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();

    // ---- partial sums: accumulator element i of a thread = tile row 16 * warp + lane / 4 + 8 * ((i / 2) % 2) (+ 64 in acc1),
    //      column 8 * (i / 4) + 2 * (lane % 4) + i % 2; rows past M and columns past N (other groups' channels) are dropped.
    float* out = P.out + (int64_t)split * P.slice_stride + ((int64_t)g * P.T + t) * P.M * P.N;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const float* acc = h ? acc1 : acc0;
#pragma unroll
        for (int i = 0; i < BN / 2; i += 2) {
            const int m = mt * kBM + 64 * h + 16 * warp + (lane >> 2) + 8 * ((i >> 1) & 1);
            const int n = nt * BN + 8 * (i >> 2) + 2 * (lane & 3);
            if (m < P.M && n < P.N) *reinterpret_cast<float2*>(out + (int64_t)m * P.N + n) = make_float2(acc[i], acc[i + 1]);
        }
    }
}

// dw = partial[0] + partial[1] + ... in slice order.
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float4* __restrict__ partial, int splits, int64_t stride4, int64_t n4,
                                                           float4* __restrict__ dw) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 a = partial[i];
        for (int s = 1; s < splits; ++s) {
            const float4 b = partial[(int64_t)s * stride4 + i];
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        dw[i] = a;
    }
}

// Channel-major operand of n3d_conv_wgrad (see the header).
__global__ void __launch_bounds__(256) wgrad_operand_kernel(const float* __restrict__ x, int64_t xs0, int64_t xs1, int64_t xs2, int64_t xs3,
                                                            int N, int C, int H, int W, int s, int pt, int pl, int PH, int PW, int shift,
                                                            int64_t ld, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    const int64_t used = (int64_t)s * s * N * PH * PW, total = (int64_t)C * ld;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = idx / ld, j = idx - c * ld + shift;
        float v = 0.f;
        if (j >= 0 && j < used) {
            const int px = (int)(j % PW);
            int64_t r = j / PW;
            const int py = (int)(r % PH);
            r /= PH;
            const int n = (int)(r % N), par = (int)(r / N);
            const int iy = s * (py - pt) + par / s, ix = s * (px - pl) + par % s;
            if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg(x + n * xs0 + c * xs1 + iy * xs2 + ix * xs3);
        }
        split_bf16(v, hi[idx], lo[idx]);
    }
}

// 2-D bf16 tensor [rows][cols] with row stride ld elements, box = 64 columns x box_rows rows, SWIZZLE_128B, zero fill outside.
int make_tmap_2d(CUtensorMap* tm, const void* base, int64_t cols, int64_t rows, int64_t ld, int box_rows) {
    const uint64_t dims[2] = {(uint64_t)cols, (uint64_t)rows}, stride = (uint64_t)ld * 2;
    const uint32_t box[2] = {(uint32_t)kBK, (uint32_t)box_rows};
    return n3d_encode_tmap(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, 2, dims, &stride, box, CU_TENSOR_MAP_SWIZZLE_128B, "n3d_conv_wgrad");
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }
}  // namespace

extern "C" int n3d_conv_wgrad(const N3DConvWgrad* p, void* stream) {
    N3D_CHECK_ARG(p, "n3d_conv_wgrad: null descriptor");
    N3D_CHECK_ARG(p->a_hi && p->a_lo && p->b_hi && p->b_lo && p->dw, "n3d_conv_wgrad: null operand or output");
    N3D_CHECK_ARG(p->G >= 1 && p->G <= 65535 && p->M >= 1 && p->N >= 8 && p->N % 8 == 0, "n3d_conv_wgrad: bad sizes G %d, M %d, N %d (N a multiple of 8)",
                  p->G, p->M, p->N);
    N3D_CHECK_ARG(p->T >= 1 && p->T <= 9, "n3d_conv_wgrad: %d taps", p->T);
    N3D_CHECK_ARG(p->K >= kBK && p->K % kBK == 0 && p->K <= (1ll << 30), "n3d_conv_wgrad: K must be a positive multiple of 64 up to 2^30");
    N3D_CHECK_ARG(p->lda % 8 == 0 && p->ldb % 8 == 0 && p->a_cols >= 1 && p->a_cols <= p->lda && p->b_cols >= 1 && p->b_cols <= p->ldb &&
                  p->a_cols < (1ll << 31) && p->b_cols < (1ll << 31), "n3d_conv_wgrad: bad operand geometry (row strides are multiples of 8 elements)");
    for (int t = 0; t < p->T; ++t)
    {
        N3D_CHECK_ARG(p->a_off[t] > -(1ll << 30) && p->a_off[t] < (1ll << 30) && p->b_off[t] > -(1ll << 30) && p->b_off[t] < (1ll << 30),
                      "n3d_conv_wgrad: tap %d offset out of range", t);
        N3D_CHECK_ARG(p->a_off[t] % 8 == 0 && p->b_off[t] % 8 == 0, "n3d_conv_wgrad: tap %d column offsets must be multiples of 8 (16-byte TMA boxes)", t);
        N3D_CHECK_ARG(p->a_row[t] >= 0 && p->b_row[t] >= 0 && p->a_row[t] + (int64_t)p->G * p->M <= p->a_rows &&
                      p->b_row[t] + (int64_t)p->G * p->N <= p->b_rows, "n3d_conv_wgrad: tap %d rows past the operands' rows", t);
    }
    const int ksteps = (int)(p->K / kBK);
    N3D_CHECK_ARG(p->splits >= 1 && p->splits <= ksteps, "n3d_conv_wgrad: %d K slices for %d K steps", p->splits, ksteps);
    N3D_CHECK_ARG(p->splits == 1 || p->partial, "n3d_conv_wgrad: split-K needs the partial-sum workspace");
    N3D_CHECK_ARG(aligned16(p->a_hi) && aligned16(p->a_lo) && aligned16(p->b_hi) && aligned16(p->b_lo) && aligned16(p->dw) && aligned16(p->partial),
                  "n3d_conv_wgrad: operands, partial and dw must be 16-byte aligned");
    const int bn = p->N <= 32 ? 32 : p->N <= 64 ? 64 : 128;
    const int m_tiles = n3d_div_up(p->M, kBM), n_tiles = n3d_div_up(p->N, bn);
    N3D_CHECK_ARG((int64_t)m_tiles * n_tiles * p->splits < (1ll << 31), "n3d_conv_wgrad: too many tiles");

    WParams P;
    memset(&P, 0, sizeof(P));
    P.G = p->G; P.M = p->M; P.N = p->N; P.T = p->T; P.splits = p->splits; P.n_tiles = n_tiles; P.ksteps = ksteps;
    for (int t = 0; t < p->T; ++t) {
        P.a_off[t] = (int)p->a_off[t]; P.b_off[t] = (int)p->b_off[t]; P.a_row[t] = p->a_row[t]; P.b_row[t] = p->b_row[t];
    }
    P.stage_bytes = 2 * kABytes + 2 * bn * kBK * 2;
    P.stages = min(kMaxStages, kRingBytes / P.stage_bytes);
    const int64_t slab = (int64_t)p->G * p->T * p->M * p->N;
    P.out = p->splits > 1 ? p->partial : p->dw;
    P.slice_stride = slab;
    int rc;
    if ((rc = make_tmap_2d(&P.tmA[0], p->a_hi, p->a_cols, p->a_rows, p->lda, kBM)) != N3D_OK) return rc;
    if ((rc = make_tmap_2d(&P.tmA[1], p->a_lo, p->a_cols, p->a_rows, p->lda, kBM)) != N3D_OK) return rc;
    if ((rc = make_tmap_2d(&P.tmB[0], p->b_hi, p->b_cols, p->b_rows, p->ldb, bn)) != N3D_OK) return rc;
    if ((rc = make_tmap_2d(&P.tmB[1], p->b_lo, p->b_cols, p->b_rows, p->ldb, bn)) != N3D_OK) return rc;

    typedef void (*WgradKernel)(const WParams);
    const WgradKernel kern = bn == 32 ? conv_wgrad_kernel<32> : bn == 64 ? conv_wgrad_kernel<64> : conv_wgrad_kernel<128>;
    const int smem = P.stages * P.stage_bytes + 16 * P.stages + 1024;
    if ((rc = n3d_smem_optin((const void*)kern, smem, "n3d_conv_wgrad")) != N3D_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    kern<<<dim3(m_tiles * n_tiles * p->splits, p->T, p->G), kThreads, smem, st>>>(P);
    N3D_CHECK_LAUNCH("n3d_conv_wgrad");
    if (p->splits > 1) {
        wgrad_reduce_kernel<<<n3d_grid(slab / 4, 256), 256, 0, st>>>((const float4*)p->partial, p->splits, slab / 4, slab / 4, (float4*)p->dw);
        N3D_CHECK_LAUNCH("n3d_conv_wgrad (split-K reduction)");
    }
    return N3D_OK;
}

extern "C" int n3d_wgrad_operand(const float* x, const int64_t x_strides[4], int N, int C, int H, int W, int s, int pt, int pl, int PH, int PW,
                                 int shift, int64_t ld, void* hi, void* lo, void* stream) {
    N3D_CHECK_ARG(x && x_strides && hi && lo, "n3d_wgrad_operand: null pointer");
    N3D_CHECK_ARG(N >= 1 && C >= 1 && H >= 1 && W >= 1 && PH >= 1 && PW >= 1 && (s == 1 || s == 2), "n3d_wgrad_operand: bad sizes");
    N3D_CHECK_ARG(ld % 8 == 0 && ld >= (int64_t)s * s * N * PH * PW, "n3d_wgrad_operand: row stride %lld must be a multiple of 8 and hold s^2 N PH PW = %lld columns",
                  (long long)ld, (long long)s * s * N * PH * PW);
    N3D_CHECK_ARG(aligned16(hi) && aligned16(lo), "n3d_wgrad_operand: hi and lo must be 16-byte aligned");
    wgrad_operand_kernel<<<n3d_grid((int64_t)C * ld, 256, 16), 256, 0, (cudaStream_t)stream>>>(
        x, x_strides[0], x_strides[1], x_strides[2], x_strides[3], N, C, H, W, s, pt, pl, PH, PW, shift, ld, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
    N3D_CHECK_LAUNCH("n3d_wgrad_operand");
    return N3D_OK;
}
