// Fused volume renderer for sm_90a, warp-specialised: ray generation, stratified depths, tri-plane bilinear fetch (+ mean over
// planes), MLP decoder (32 -> 64 softplus -> 1 + 32, sigmoid) on tensor cores, coarse compositing weights, importance
// resampling, sort-merge of coarse + fine samples and final alpha compositing in ONE persistent kernel.  Replaces
// RaySampler.forward (ray_sampler.py:24-63), ImportanceRenderer.forward (renderer.py:95-268), OSGDecoder.forward
// (triplane_next3d.py:359-371) and MipRayMarcher2.run_forward (ray_marcher.py:27-66).
//
// One CTA per SM, 16 warps:
//   warps  0-7   E ("epilogue") : two sets of four; warp w owns tile rows 32*(w%4).., set s = w/4 owns hidden units 32s..32s+31 and
//                colour channels 16s..16s+15.  Each E warp runs its own share of the decoder on tensor cores (mma.sync m16n8k16,
//                bf16x3 = hi*hi + hi*lo + lo*hi, fp32 accumulate); the two warps of a row quarter exchange the hidden layer through
//                shared memory.  For the per-ray phases, thread = tile row = one depth sample of one ray in every tile of its group.
//   warps  8-15  G ("gather")   : build the layer-1 A operand in shared memory; work item = 32 rows (a quarter) of a tile, items
//                dealt round-robin to the eight warps; 12 bilinear taps per sample fetched as 128-bit loads, 8 lanes x 4
//                channels per sample.
// Work unit: a GROUP = 128/L rays (a 4x2, 2x2 or 1x2 pixel block) x L lanes each, L = 16 (<= 48 samples per pass), 32 (<= 96)
// or 64 (<= 192).  A pass of a group is T = ceil(D / L) <= 3 tiles of 128 rows; row = ray_slot * L + j holds sample k = tile * L + j
// of that ray, so a ray's samples always sit in the same L lanes and every per-ray phase (transmittance scan, PDF/CDF,
// inverse-CDF sampling, rank merge, weighted colour sum) runs on registers + warp shuffles, no CTA-wide barrier anywhere.  At
// L = 64 a ray spans the two warps 2r, 2r + 1 of one E set; the steps that cross the warp boundary (scan carries, sums, the
// neighbour sample, the merge's bucket prefix) exchange a few words through shared memory under a 64-thread named barrier.
// Tile stream of a CTA: C(0) | C(1) F(0) | C(2) F(1) | ...  (coarse tiles of group r+1 are issued before the fine tiles of
// group r, so the importance sampling of a group never stalls the gather warps).
//
// Colour slots: nine tiles of sigmoid colours (coarse of two groups + fine of one) wait in shared memory until the final weights
// are known, stored as 16-bit unsigned normalised values (absolute error <= 2^-17, below the fp32 decoder's own error after
// compositing); then each thread accumulates coefficient x colour for its own rows.
#include "common.cuh"
#include "tc_ptx.cuh"
#include "render_common.cuh"

namespace {
using namespace n3d_tc;
using namespace n3d_rc;

constexpr int kEWarps = 8, kGWarps = 8;
constexpr int kWarps = kEWarps + kGWarps;
constexpr int kThreads = kWarps * 32;           // 512 (16 warps -> 128 registers per thread)
constexpr int kMaxT = 3;                        // tiles per pass
constexpr unsigned FULL = 0xffffffffu;

// shared-memory byte offsets (base 1024-aligned)
constexpr int kOffW0hi = 0, kOffW0lo = 4096, kOffWchi = 8192, kOffWclo = 12288, kOffWshi = 16384, kOffWslo = 18432;
constexpr int kNF = 2;                                          // layer-1 A-operand buffers
constexpr int kOffF = 20480;                                    // kNF x (hi 8 KiB | lo 8 KiB)
constexpr int kOffTaps = kOffF + kNF * 16384;                   // 8 warps x [12][32] x (offset, weight)
constexpr int kTapBytesPerWarp = 12 * 32 * 8;
constexpr int kOffEscr = kOffTaps + kGWarps * kTapBytesPerWarp; // per-E-warp scratch
constexpr int kEscrFloats = 960;
constexpr int kOffTfine = kOffEscr + kEWarps * kEscrFloats * 4; // [2][rays per group][Df] fine depths for the gather warps
constexpr int kTfineFloats = 384;
constexpr int kHStride = 36;                                    // 32-bit words per row of the hidden buffer (32 bf16 pairs + pad)
constexpr int kOffH = kOffTfine + 2 * kTfineFloats * 4;         // hidden layer [128][kHStride] bf16x2 words: hi | lo
constexpr int kOffSig = kOffH + 2 * 128 * kHStride * 4;         // [2][128] raw sigma of the last two tiles
constexpr int kNumSlots = 9;
constexpr int kOffCol = kOffSig + 2 * 128 * 4;                  // kNumSlots x [128][32] unorm16 sigmoid colours
constexpr int kOffBias = kOffCol + kNumSlots * 128 * 64;        // b0 * log2e [64] | b1 colour [32] | b1 sigma [1] (+pad)
constexpr int kOffBar = kOffBias + (64 + 32 + 16) * 4;
constexpr int kNumBars = 2 * kNF + 2;
constexpr int kSmemBytes = kOffBar + kNumBars * 8;

enum { BAR_FFULL = 0, BAR_FEMPTY = kNF, BAR_FINE = 2 * kNF };

struct FusedK {
    N3DRender p;
    int M;                       // rays per image
    float delta_coarse, scale;
    int Tc, Tf;                  // tiles per coarse / fine pass
    int gw, log2gw;              // pixel block of a group: gw x 2
    int blocks_x, gpi;           // group map: blocks of 4 x 8 groups, groups per image (padded)
    long long total_groups;
    float* samples;              // render_fused_kernel<L, true>: per ray the D sorted depths, then the D - 1 final weights
};

// ---------------------------------------------------------------------------------------------------------------- group -> rays
struct RayId {
    int n, row, col;
    bool ok;
    long long gr;
};
__device__ __forceinline__ RayId ray_of(const FusedK& K, int gg, int rs) {
    RayId r;
    const int n = gg / K.gpi;
    const int q = gg - n * K.gpi;
    const int blk = q >> 5, inb = q & 31;
    const int byi = blk / K.blocks_x, bxi = blk - byi * K.blocks_x;
    const int tx = bxi * 4 + (inb & 3), ty = byi * 8 + (inb >> 2);
    r.col = tx * K.gw + (rs & (K.gw - 1));
    r.row = ty * 2 + (rs >> K.log2gw);
    r.n = n;
    r.ok = r.col < K.p.res && r.row < K.p.res;
    r.gr = (long long)n * K.M + (long long)r.row * K.p.res + r.col;
    return r;
}

struct Ray {
    float ox, oy, oz, dx, dy, dz;
    uint32_t img4;
    long long gr;
    bool ok;
};
// ray_sampler.py:43-63 for the ray in slot rs of group gg
__device__ __forceinline__ Ray make_ray(const FusedK& K, int gg, int rs) {
    const N3DRender& P = K.p;
    const RayId id = ray_of(K, gg, rs);
    Ray r;
    r.ok = id.ok;
    r.gr = id.gr;
    r.img4 = (uint32_t)(id.n / P.views) * (uint32_t)(3 * P.PH * P.PW * 128);       // byte offset of the image's plane set
    r.ox = r.oy = r.oz = r.dx = r.dy = r.dz = 0.f;
    if (id.ok) {
        float o[3], d[3];
        camera_ray(P, id.n, id.row, id.col, o, d);
        r.ox = o[0]; r.oy = o[1]; r.oz = o[2];
        r.dx = d[0]; r.dy = d[1]; r.dz = d[2];
    }
    return r;
}

__device__ __forceinline__ float coarse_depth(const FusedK& K, uint64_t seed, long long gr, int k) {
    const N3DRender& P = K.p;
    const float u = P.u_coarse ? __ldg(P.u_coarse + gr * P.depth_coarse + k) : hash_uniform(seed, (uint64_t)(gr * P.depth_coarse + k));
    return linspace_at(P.ray_start, P.ray_end, P.depth_coarse, k) + u * K.delta_coarse;
}

// ---------------------------------------------------------------------------------------------------------------- gather warps
// The four bilinear taps of plane pl (0 <- (x, y), 1 <- (x, z), 2 <- (z, y); grid_sample zeros padding, align_corners=False) at
// the scaled point (x, y, z): texel byte offsets, weights and the derivatives of the weights along the plane's two world axes (a, b)
// (d ix / d x_a = scale * PW / 2); the 1/3 of the plane mean is folded into all three.  Taps outside the plane and invalid samples
// get weight 0 and point at texel 0.  The renderer's gather (setup_taps) and the normal pass both take their taps from here, so a
// sample's feature is the same float expression in both kernels (the gather uses the offsets and weights only).
struct PlaneTaps {
    uint32_t off[4];
    float w[4], wa[4], wb[4];
};
__device__ __forceinline__ PlaneTaps plane_taps(int pl, float x, float y, float z, bool valid, uint32_t img4, int PH, int PW, float scale) {
    PlaneTaps t;
    const float gx = pl == 2 ? z : x, gy = pl == 1 ? z : y;
    const float ix = ((gx + 1.f) * (float)PW - 1.f) * 0.5f, iy = ((gy + 1.f) * (float)PH - 1.f) * 0.5f;
    const float flx = floorf(ix), fly = floorf(iy);
    const float fx = ix - flx, fy = iy - fly;
    const int x0 = (int)fminf(fmaxf(flx, -2.f), (float)PW), y0 = (int)fminf(fmaxf(fly, -2.f), (float)PH);
    const uint32_t pbase = img4 + (uint32_t)(pl * PH * PW) * 128u;
    const float ka = scale * (float)PW * (0.5f / 3.f), kb = scale * (float)PH * (0.5f / 3.f);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int xi = x0 + (c & 1), yi = y0 + (c >> 1);
        const float wx = (c & 1) ? fx : 1.f - fx, wy = (c >> 1) ? fy : 1.f - fy;
        const bool inside = valid && xi >= 0 && xi < PW && yi >= 0 && yi < PH;
        t.off[c] = inside ? pbase + (uint32_t)(yi * PW + xi) * 128u : 0u;
        t.w[c] = inside ? wx * wy * (1.f / 3.f) : 0.f;
        t.wa[c] = inside ? ((c & 1) ? wy : -wy) * ka : 0.f;
        t.wb[c] = inside ? ((c >> 1) ? wx : -wx) * kb : 0.f;
    }
    return t;
}

// 12 bilinear taps of one sample (3 planes x 4 corners) into `taps`: byte offset of the texel + weight / 3.
__device__ __forceinline__ void setup_taps(uint2* __restrict__ taps, int lane, float px, float py, float pz, bool valid, uint32_t img4, int PH, int PW,
                                           float scale) {
    const float x = scale * px, y = scale * py, z = scale * pz;
#pragma unroll
    for (int pl = 0; pl < 3; ++pl) {
        const PlaneTaps t = plane_taps(pl, x, y, z, valid, img4, PH, PW, scale);
#pragma unroll
        for (int c = 0; c < 4; ++c) taps[(pl * 4 + c) * 32 + lane] = make_uint2(t.off[c], __float_as_uint(t.w[c]));
    }
}

// 32 samples whose taps sit in `taps`: lanes = 8 samples x 4 channel octets per step (4 steps); every tap is one 256-bit load per
// lane (four lanes cover the texel's 128-byte line), accumulated with packed fp32x2 FMAs; the mean feature goes straight into the
// K-major SWIZZLE_64B bf16 (hi, lo) A-operand tile rows row0..row0+31 as one 16-byte store per lane and operand half.
// Weights already carry the 1/3 of the plane mean.
__device__ __forceinline__ void gather_rows(const float* __restrict__ planes, const uint2* __restrict__ taps, uint8_t* __restrict__ f_hi,
                                            uint8_t* __restrict__ f_lo, int row0, int lane) {
    const int c8 = lane & 3, s8 = lane >> 2;
    const char* const base = reinterpret_cast<const char*>(planes) + c8 * 32;
    const uint2* const tl = taps + s8;                          // + tap * 32 + step * 8
#pragma unroll 1
    for (int step = 0; step < 4; ++step) {
        float2 acc[4];
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            uint2 tp[6];
            float v[6][8];
#pragma unroll
            for (int i = 0; i < 6; ++i) tp[i] = tl[(half * 6 + i) * 32 + step * 8];
#pragma unroll
            for (int i = 0; i < 6; ++i) ldg_nc_256(reinterpret_cast<const float*>(base + tp[i].x), v[i]);
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                const float wt = __uint_as_float(tp[i].y);
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float2 x = make_float2(v[i][2 * c], v[i][2 * c + 1]);
                    acc[c] = (half == 0 && i == 0) ? make_float2(__fmul_rn(wt, x.x), __fmul_rn(wt, x.y))
                                                   : make_float2(__fmaf_rn(wt, x.x, acc[c].x), __fmaf_rn(wt, x.y, acc[c].y));
                }
            }
        }
        uint32_t h[4], l[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) split_bf16x2(acc[c].x, acc[c].y, h[c], l[c]);
        const uint32_t off = sw64_off(row0 + step * 8 + s8, c8 * 16);
        *reinterpret_cast<uint4*>(f_hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(f_lo + off) = make_uint4(l[0], l[1], l[2], l[3]);
    }
}

// ---------------------------------------------------------------------------------------------------------------- per-ray math
// Reduce-scatter of 16 values over the 16 (k32 = false) or 32 lanes of a warp segment: lane ends with the sum of value (lane & 15)
// in acc[0].
template <bool k32>
__device__ __forceinline__ void reduce_scatter16(float (&acc)[16], int lane) {
    if (k32) {
#pragma unroll
        for (int c = 0; c < 16; ++c) acc[c] += __shfl_xor_sync(FULL, acc[c], 16);
    }
#pragma unroll
    for (int h = 8; h >= 1; h >>= 1) {
        const bool up = (lane & h) != 0;
#pragma unroll
        for (int c = 0; c < h; ++c) {
            const float send = up ? acc[c] : acc[c + h];
            const float keep = up ? acc[c + h] : acc[c];
            acc[c] = keep + __shfl_xor_sync(FULL, send, h);
        }
    }
}

// RaySeg<L>: the lanes that hold one ray.  Sample k = t * L + j of the ray sits in register slot t of the ray's lane j, and every
// per-ray step that combines lanes is one of these methods, so the per-ray phases are written once for all three layouts.  Here
// L = 16 or 32: the L lanes [lane & ~(L-1), +L) of one warp, j = lane & (L - 1); the steps are warp shuffles.
template <int L>
struct RaySeg {
    // Scratch of the warp's kRays rays, in floats of the warp's own area: region A [0, 640) = sd | sg | wb (kRays x (Dt + 2) each),
    // aliased by the cdf during importance sampling and by the u-bucket tables during ranking; tcs at 640 (kRays x Dc), tfs at 736
    // (kRays x Df), hist at 832 (kRays x (Dc + 1)).
    static constexpr int kRays = 32 / L, kTcOff = 640, kTfOff = 736, kHistOff = 832;
    __device__ __forceinline__ static int area(int warp) { return warp; }

    int lane;
    __device__ __forceinline__ RaySeg(float*, int, int lane_) : lane(lane_) {}

    // out[t] = value of sample k + 1 (`last` after the final slot)
    template <int NT>
    __device__ __forceinline__ void next(const float (&v)[NT], float last, float (&out)[NT]) {
#pragma unroll
        for (int t = 0; t < NT; ++t) {
            const float a = __shfl_down_sync(FULL, v[t], 1);
            const float b = __shfl_sync(FULL, t + 1 < NT ? v[t + 1] : last, lane & ~(L - 1));
            out[t] = ((lane & (L - 1)) == L - 1) ? b : a;
        }
    }
    // out[t] = value of sample k - 1 (`first` before sample 0)
    template <int NT>
    __device__ __forceinline__ void prev(const float (&v)[NT], float first, float (&out)[NT]) {
#pragma unroll
        for (int t = 0; t < NT; ++t) {
            const float a = __shfl_up_sync(FULL, v[t], 1);
            const float b = __shfl_sync(FULL, t > 0 ? v[t - 1] : first, lane | (L - 1));
            out[t] = ((lane & (L - 1)) == 0) ? b : a;
        }
    }
    // sum over the ray: the same bits in every lane of it
    __device__ __forceinline__ float sum(float v) {
#pragma unroll
        for (int o = L / 2; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
        return v;
    }
    // inclusive scan (product when MUL) in sample order
    template <bool MUL, int NT>
    __device__ __forceinline__ void scan(float (&x)[NT]) {
        float carry = MUL ? 1.f : 0.f;
        const int j = lane & (L - 1);
#pragma unroll
        for (int t = 0; t < NT; ++t) {
            float v = x[t];
#pragma unroll
            for (int o = 1; o < L; o <<= 1) {
                const float up = __shfl_up_sync(FULL, v, o);
                if (j >= o) v = MUL ? v * up : v + up;
            }
            v = MUL ? v * carry : v + carry;
            x[t] = v;
            carry = __shfl_sync(FULL, v, lane | (L - 1));
        }
    }
    // inclusive prefix sum of one integer per lane, in lane order
    __device__ __forceinline__ int prefix(int v) {
        const int j = lane & (L - 1);
#pragma unroll
        for (int o = 1; o < L; o <<= 1) { const int up = __shfl_up_sync(FULL, v, o); if (j >= o) v += up; }
        return v;
    }
    __device__ __forceinline__ bool any(bool p) { return __any_sync(FULL, p); }
    __device__ __forceinline__ void sync() { __syncwarp(); }
    // start of a per-ray phase: nothing to wait for, the ray's lanes finished the previous phase together
    __device__ __forceinline__ void enter() {}
    // the value of lane j = 0 (read on j = 0 only)
    __device__ __forceinline__ float lead(float v) { return __shfl_sync(FULL, v, lane & ~(L - 1)); }
    // colour reduce-scatter: lane j ends with channel (j & 15) summed over the ray's lanes, in acc[0]
    __device__ __forceinline__ void reduce16(float (&acc)[16]) { reduce_scatter16<L == 32>(acc, lane); }
};

// L = 64: the two warps 2r, 2r + 1 of one E set, half h = warp & 1 holding j = 32 h + lane.  The steps that cross the warp boundary
// exchange a few words through the pair's scratch under the pair's 64-thread named barrier.  Every exchange writes one of two
// ping-pong buffers and passes the barrier once; a buffer is rewritten only after the partner has passed the next barrier, i.e.
// after it read the buffer's previous contents.  Each per-ray phase starts at the barrier, so neither warp overwrites scratch its
// partner still reads.
template <>
struct RaySeg<64> {
    // Scratch of the ray: the pair's two areas, 1920 floats: region A [0, 1160) (3 x 386; 2 x 512 bucket words), tcs at 1160, tfs at
    // 1352, hist at 1544 (193), the exchange words at 1752 (2 x 32).
    static constexpr int kRays = 1, kTcOff = 1160, kTfOff = 1352, kHistOff = 1544, kXOff = 1752;
    __device__ __forceinline__ static int area(int warp) { return warp & ~1; }

    float* words;                // 2 x 32 exchange words
    int lane, bar, h, ph;        // named barrier id (5 .. 8), warp half, current buffer
    __device__ __forceinline__ RaySeg(float* es, int warp, int lane_) : words(es + kXOff), lane(lane_), bar(5 + (warp >> 1)), h(warp & 1), ph(0) {}

    __device__ __forceinline__ float* buf() {
        float* const b = words + 32 * ph;
        ph ^= 1;
        return b;
    }
    template <int NT>
    __device__ __forceinline__ void next(const float (&v)[NT], float last, float (&out)[NT]) {
        float* const b = buf();
        if (lane == 0) {
#pragma unroll
            for (int t = 0; t < NT; ++t) b[8 * h + t] = h ? v[t] : (t + 1 < NT ? v[t + 1] : last);
        }
        sync();
#pragma unroll
        for (int t = 0; t < NT; ++t) {
            const float a = __shfl_down_sync(FULL, v[t], 1);
            out[t] = lane == 31 ? b[8 * (h ^ 1) + t] : a;
        }
    }
    template <int NT>
    __device__ __forceinline__ void prev(const float (&v)[NT], float first, float (&out)[NT]) {
        float* const b = buf();
        if (lane == 31) {
#pragma unroll
            for (int t = 0; t < NT; ++t) b[8 * h + t] = h ? (t > 0 ? v[t - 1] : first) : v[t];
        }
        sync();
#pragma unroll
        for (int t = 0; t < NT; ++t) {
            const float a = __shfl_up_sync(FULL, v[t], 1);
            out[t] = lane == 0 ? b[8 * (h ^ 1) + t] : a;
        }
    }
    __device__ __forceinline__ float sum(float v) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
        float* const b = buf();
        if (lane == 0) b[h] = v;
        sync();
        return b[0] + b[1];                                          // same order in both halves: both get the same bits
    }
    template <bool MUL, int NT>
    __device__ __forceinline__ void scan(float (&x)[NT]) {
#pragma unroll
        for (int t = 0; t < NT; ++t) {
            float v = x[t];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float up = __shfl_up_sync(FULL, v, o);
                if (lane >= o) v = MUL ? v * up : v + up;
            }
            x[t] = v;
        }
        float* const b = buf();
        if (lane == 31) {
#pragma unroll
            for (int t = 0; t < NT; ++t) b[8 * h + t] = x[t];
        }
        sync();
        float carry = MUL ? 1.f : 0.f;
#pragma unroll
        for (int t = 0; t < NT; ++t) {
            const float c1 = MUL ? carry * b[t] : carry + b[t];      // carry into half 1 of slot t
            x[t] = MUL ? x[t] * (h ? c1 : carry) : x[t] + (h ? c1 : carry);
            carry = MUL ? c1 * b[8 + t] : c1 + b[8 + t];
        }
    }
    __device__ __forceinline__ int prefix(int v) {                  // counts <= 192: exact in fp32
        float f[1] = {(float)v};
        scan<false>(f);
        return (int)f[0];
    }
    __device__ __forceinline__ bool any(bool p) {
        int r;
        asm volatile("{\n\t.reg .pred a, b;\n\tsetp.ne.s32 a, %1, 0;\n\tbar.red.or.pred b, %2, 64, a;\n\tselp.s32 %0, 1, 0, b;\n\t}"
                     : "=r"(r) : "r"((int)p), "r"(bar) : "memory");
        return r != 0;
    }
    __device__ __forceinline__ void sync() { asm volatile("bar.sync %0, 64;" ::"r"(bar) : "memory"); }
    __device__ __forceinline__ void enter() { sync(); }
    __device__ __forceinline__ float lead(float v) { return v; }     // j = 0 is lane 0 of half 0 itself
    __device__ __forceinline__ void reduce16(float (&acc)[16]) {
        reduce_scatter16<true>(acc, lane);
        float* const b = buf();                                      // half 1's channel sums join half 0's (j = lane < 16)
        if (h == 1 && lane < 16) b[lane] = acc[0];
        sync();
        if (h == 0 && lane < 16) acc[0] += b[lane];
    }
};

// MipRayMarcher2 weights (ray_marcher.py:27-46) of a depth-sorted list of `cnt` samples (d, sg):
//   alpha_k = 1 - exp(-softplus((s_k + s_k+1)/2 - 1) * (t_k+1 - t_k)),  T_k = prod_{i<k} (1 - alpha_i + 1e-10),  w_k = alpha_k T_k
// w_k = 0 for k >= cnt - 1.  tmid_k = (t_k + t_k+1) / 2.  j: the lane's index in the ray.
template <int L, int NT>
__device__ __forceinline__ void march_weights(RaySeg<L>& seg, const float (&d)[NT], const float (&sg)[NT], int cnt, int j, float (&w)[NT],
                                              float (&tmid)[NT]) {
    float dn[NT], sn[NT], fac[NT], al[NT], ex[NT];
    seg.next(d, 0.f, dn);
    seg.next(sg, 0.f, sn);
#pragma unroll
    for (int t = 0; t < NT; ++t) {
        const int k = t * L + j;
        float alpha = 0.f;
        if (k < cnt - 1) {
            const float delta = dn[t] - d[t];
            const float dens = softplus_fast((sg[t] + sn[t]) * 0.5f - 1.f);
            // 1 - exp(-x): the MUFU exponential is ~2e-7 off near 1, a BIAS that adds up over ~190 thin intervals; below 1/16 the
            // alternating series is exact to 1e-8 relative
            const float xx = dens * delta;
            const float ser = xx * (1.f - xx * (0.5f - xx * (0.16666667f - xx * (0.041666668f - xx * 0.0083333338f))));
            alpha = xx < 0.0625f ? ser : 1.f - ex2_approx(-kLog2e * xx);
        }
        al[t] = alpha;
        fac[t] = k < cnt - 1 ? (1.f - alpha + 1e-10f) : 1.f;
        tmid[t] = (d[t] + dn[t]) * 0.5f;
    }
    seg.template scan<true>(fac);
    seg.prev(fac, 1.f, ex);
#pragma unroll
    for (int t = 0; t < NT; ++t) w[t] = al[t] * ((t == 0 && j == 0) ? 1.f : ex[t]);
}

// Tile stream of a CTA with n groups: C(0) | C(1) F(0) | ... | C(n-1) F(n-2) | F(n-1); every role walks it with the same iterator.
struct TileIter {
    int n, Tc, Tf;
    int r, kind, t;                 // round, 0 coarse / 1 fine, tile of the pass
    __device__ __forceinline__ TileIter(int n_, int Tc_, int Tf_) : n(n_), Tc(Tc_), Tf(Tf_), r(0), kind(0), t(-1) {}
    __device__ __forceinline__ bool next() {
        ++t;
        for (;;) {
            if (kind == 0) {
                if (r < n && t < Tc) return true;
                kind = 1; t = 0;
            }
            if (r >= 1 && t < Tf) return true;
            kind = 0; t = 0; ++r;
            if (r > n) return false;
        }
    }
    __device__ __forceinline__ int group() const { return kind == 0 ? r : r - 1; }
};

struct Smem {
    uint8_t* base;
    __device__ __forceinline__ uint32_t bar(int i) const { return smem_u32(base + kOffBar + i * 8); }
};

// Gather warp: fill rows row0 .. row0 + 31 of A buffer i % kNF (the i-th tile) from the taps the warp just wrote, once the
// epilogue has freed the buffer, and publish them.
__device__ __forceinline__ void fill_buffer(const Smem& S, const float* __restrict__ planes, const uint2* __restrict__ taps, int i, int row0,
                                            int lane) {
    __syncwarp();
    const int b = i % kNF;
    if (i >= kNF) mbar_wait_sleep(S.bar(BAR_FEMPTY + b), (uint32_t)((i / kNF - 1) & 1), 40u);
    gather_rows(planes, taps, S.base + kOffF + b * 16384, S.base + kOffF + b * 16384 + 8192, row0, lane);
    __syncwarp();
    if (lane == 0) mbar_arrive(S.bar(BAR_FFULL + b));
}

// Decoder weights -> bf16 (hi, lo) B-operand tiles in shared memory, with the activation scalings folded in: layer 1 produces
// x * log2(e); hidden units are kept as softplus / ln2; colour logits as -(x) * log2(e) (the argument of ex2 in the sigmoid).
__device__ __forceinline__ void stage_decoder(uint8_t* sb, const float* __restrict__ w0, const float* __restrict__ b0, const float* __restrict__ w1,
                                              const float* __restrict__ b1, int tid) {
    float* const sB0 = reinterpret_cast<float*>(sb + kOffBias);
    float* const sB1c = sB0 + 64;
    float* const sB1s = sB1c + 32;
    for (int i = tid; i < kHidden * kFeat; i += kThreads) {               // W0 [64][32]: row = hidden unit, K = 32 (SWIZZLE_64B)
        const int n = i / kFeat, k = i - n * kFeat;
        __nv_bfloat16 h, l;
        split_bf16(__ldg(w0 + i) * kLog2e, h, l);        // layer 1 produces x * log2(e) (the argument of ex2)
        *reinterpret_cast<__nv_bfloat16*>(sb + kOffW0hi + sw64_off(n, k * 2)) = h;
        *reinterpret_cast<__nv_bfloat16*>(sb + kOffW0lo + sw64_off(n, k * 2)) = l;
    }
    for (int i = tid; i < 32 * kHidden; i += kThreads) {                  // colour rows of W1 (outputs 1..32) [32][64] (SWIZZLE_128B)
        const int n = i / kHidden, k = i - n * kHidden;
        __nv_bfloat16 h, l;
        split_bf16(-__ldg(w1 + (n + 1) * kHidden + k), h, l);   // hidden units are kept as softplus / ln2; colour logits as -x * log2(e)
        *reinterpret_cast<__nv_bfloat16*>(sb + kOffWchi + sw128_off(n, k * 2)) = h;
        *reinterpret_cast<__nv_bfloat16*>(sb + kOffWclo + sw128_off(n, k * 2)) = l;
    }
    for (int i = tid; i < 16 * kHidden; i += kThreads) {                  // sigma row of W1 (output 0) padded to N = 16
        const int n = i / kHidden, k = i - n * kHidden;
        __nv_bfloat16 h, l;
        split_bf16(n == 0 ? __ldg(w1 + k) * kLn2 : 0.f, h, l);
        *reinterpret_cast<__nv_bfloat16*>(sb + kOffWshi + sw128_off(n, k * 2)) = h;
        *reinterpret_cast<__nv_bfloat16*>(sb + kOffWslo + sw128_off(n, k * 2)) = l;
    }
    for (int i = tid; i < kHidden; i += kThreads) sB0[i] = __ldg(b0 + i) * kLog2e;
    for (int i = tid; i < 32; i += kThreads) sB1c[i] = -kLog2e * __ldg(b1 + 1 + i);
    if (tid == 0) sB1s[0] = __ldg(b1);
}

__device__ __forceinline__ uint32_t lds32(const uint8_t* p) { return *reinterpret_cast<const uint32_t*>(p); }

// Layer 1 of tile ti for E warp (q, eset): rows 32q..32q+31 x hidden units 32 eset..+31 = [32 x 32] x [32 x 32], bf16x3 on mma.sync;
// frees the A buffer, then softplus -> bf16 (hi, lo) words -> hidden buffer, and waits for the partner warp's half of the rows.
// hidden unit / ln2 = max(log2(1 + 2^min(y, 126)), y) with y = (x + b0) * log2(e): exact softplus for every finite input (for
// y > 24 the sum rounds to 2^y); ln2 is folded into the layer-2 weights.
__device__ __forceinline__ void layer1_tile(const Smem& S, int q, int eset, int lane, int ti) {
    uint8_t* const sb = S.base;
    const int b = ti % kNF;
    mbar_wait_sleep(S.bar(BAR_FFULL + b), (uint32_t)((ti / kNF) & 1), 20u);
    const uint8_t* const fh = sb + kOffF + b * 16384;
    const uint8_t* const fl = fh + 8192;
    const int g = lane >> 2, c = lane & 3;
    float acc[2][4][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;
#pragma unroll
    for (int ks = 0; ks < kFeat / 16; ++ks) {
        uint32_t bh[4][2], bl[4][2];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const int n = 32 * eset + 8 * nt + g;
            bh[nt][0] = lds32(sb + kOffW0hi + sw64_off(n, ks * 32 + 4 * c)); bh[nt][1] = lds32(sb + kOffW0hi + sw64_off(n, ks * 32 + 16 + 4 * c));
            bl[nt][0] = lds32(sb + kOffW0lo + sw64_off(n, ks * 32 + 4 * c)); bl[nt][1] = lds32(sb + kOffW0lo + sw64_off(n, ks * 32 + 16 + 4 * c));
        }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            const int r = 32 * q + 16 * mt + g;
            uint32_t ah[4], al[4];
            ah[0] = lds32(fh + sw64_off(r, ks * 32 + 4 * c)); ah[1] = lds32(fh + sw64_off(r + 8, ks * 32 + 4 * c));
            ah[2] = lds32(fh + sw64_off(r, ks * 32 + 16 + 4 * c)); ah[3] = lds32(fh + sw64_off(r + 8, ks * 32 + 16 + 4 * c));
            al[0] = lds32(fl + sw64_off(r, ks * 32 + 4 * c)); al[1] = lds32(fl + sw64_off(r + 8, ks * 32 + 4 * c));
            al[2] = lds32(fl + sw64_off(r, ks * 32 + 16 + 4 * c)); al[3] = lds32(fl + sw64_off(r + 8, ks * 32 + 16 + 4 * c));
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                mma_bf16_16816(acc[mt][nt], ah, bh[nt][0], bh[nt][1]);
                mma_bf16_16816(acc[mt][nt], ah, bl[nt][0], bl[nt][1]);
                mma_bf16_16816(acc[mt][nt], al, bh[nt][0], bh[nt][1]);
            }
        }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(S.bar(BAR_FEMPTY + b));
    const float* const sB0 = reinterpret_cast<const float*>(sb + kOffBias);
    uint32_t* const Hh = reinterpret_cast<uint32_t*>(sb + kOffH);
    uint32_t* const Hl = Hh + 128 * kHStride;
    float y[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) y[i] = acc[i >> 4][(i >> 2) & 3][i & 3] + sB0[32 * eset + 8 * ((i >> 2) & 3) + 2 * c + (i & 1)];
    // explicit stages over the 32 independent values: the MUFU operations issue back to back instead of one dependent chain per value
    float e[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) e[i] = ex2_approx(fminf(y[i], 126.f));
#pragma unroll
    for (int i = 0; i < 32; ++i) e[i] = lg2_approx(1.f + e[i]);
#pragma unroll
    for (int i = 0; i < 32; ++i) y[i] = fmaxf(e[i], y[i]);
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
        const int mt = i >> 4, nt = (i >> 2) & 3, hr = (i >> 1) & 1;
        const int row = 32 * q + 16 * mt + g + 8 * hr, word = 16 * eset + 4 * nt + c;
        uint32_t h, l;
        split_bf16x2(y[i], y[i + 1], h, l);
        Hh[row * kHStride + word] = h;
        Hl[row * kHStride + word] = l;
    }
    asm volatile("bar.sync %0, 64;" ::"r"(1 + q) : "memory");       // both halves of the quarter's hidden rows written
}

// Layer 2 of the quarter's rows from the hidden buffer: colour logits of this set's 16 channels ([32 x 64] x [64 x 16]) when
// `colours`, and (set 0) the sigma logit ([32 x 64] x [64 x 8], output 0 used).  Fragment layout of mma.m16n8k16's accumulator.
__device__ __forceinline__ void layer2_tile(const Smem& S, int q, int eset, int lane, bool colours, float (&col)[2][2][4], float (&sig)[2][4]) {
    uint8_t* const sb = S.base;
    const uint32_t* const Hh = reinterpret_cast<const uint32_t*>(sb + kOffH);
    const uint32_t* const Hl = Hh + 128 * kHStride;
    const int g = lane >> 2, c = lane & 3;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int e = 0; e < 4; ++e) { sig[mt][e] = 0.f; col[mt][0][e] = 0.f; col[mt][1][e] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < kHidden / 16; ++ks) {
        uint32_t ah[2][4], al[2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            const int r = 32 * q + 16 * mt + g;
            ah[mt][0] = Hh[r * kHStride + ks * 8 + c]; ah[mt][1] = Hh[(r + 8) * kHStride + ks * 8 + c];
            ah[mt][2] = Hh[r * kHStride + ks * 8 + 4 + c]; ah[mt][3] = Hh[(r + 8) * kHStride + ks * 8 + 4 + c];
            al[mt][0] = Hl[r * kHStride + ks * 8 + c]; al[mt][1] = Hl[(r + 8) * kHStride + ks * 8 + c];
            al[mt][2] = Hl[r * kHStride + ks * 8 + 4 + c]; al[mt][3] = Hl[(r + 8) * kHStride + ks * 8 + 4 + c];
        }
        if (colours) {
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) {
                const int n = 16 * eset + 8 * nt + g;
                const uint32_t bh0 = lds32(sb + kOffWchi + sw128_off(n, ks * 32 + 4 * c)), bh1 = lds32(sb + kOffWchi + sw128_off(n, ks * 32 + 16 + 4 * c));
                const uint32_t bl0 = lds32(sb + kOffWclo + sw128_off(n, ks * 32 + 4 * c)), bl1 = lds32(sb + kOffWclo + sw128_off(n, ks * 32 + 16 + 4 * c));
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    mma_bf16_16816(col[mt][nt], ah[mt], bh0, bh1);
                    mma_bf16_16816(col[mt][nt], ah[mt], bl0, bl1);
                    mma_bf16_16816(col[mt][nt], al[mt], bh0, bh1);
                }
            }
        }
        if (eset == 0) {
            const uint32_t bh0 = lds32(sb + kOffWshi + sw128_off(g, ks * 32 + 4 * c)), bh1 = lds32(sb + kOffWshi + sw128_off(g, ks * 32 + 16 + 4 * c));
            const uint32_t bl0 = lds32(sb + kOffWslo + sw128_off(g, ks * 32 + 4 * c)), bl1 = lds32(sb + kOffWslo + sw128_off(g, ks * 32 + 16 + 4 * c));
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                mma_bf16_16816(sig[mt], ah[mt], bh0, bh1);
                mma_bf16_16816(sig[mt], ah[mt], bl0, bl1);
                mma_bf16_16816(sig[mt], al[mt], bh0, bh1);
            }
        }
    }
}
// sigmoid of a colour logit kept as -(x + b) * log2(e)
__device__ __forceinline__ float colour_sigmoid(float z) { return rcp_approx(1.f + ex2_approx(z)); }

__device__ __forceinline__ void init_pipeline_barriers(const Smem& S) {
    for (int b = 0; b < kNF; ++b) { mbar_init(S.bar(BAR_FFULL + b), 4); mbar_init(S.bar(BAR_FEMPTY + b), kEWarps); }
}

// ---------------------------------------------------------------------------------------------------------------- the kernel
// kExport: also write every ray's merged sorted depths and final interval weights to K.samples (the input of the normal pass,
// normals_fused_kernel); nothing else changes.
template <int L, bool kExport>
__global__ void __launch_bounds__(kThreads, 1) render_fused_kernel(const __grid_constant__ FusedK K) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const N3DRender& P = K.p;
    Smem S;
    S.base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);       // pointer arithmetic keeps the shared address space
    uint8_t* const sb = S.base;
    float* const sB0 = reinterpret_cast<float*>(sb + kOffBias);         // b0 * log2(e)
    float* const sB1c = sB0 + 64;                                        // colour biases (outputs 1..32)
    float* const sB1s = sB1c + 32;                                       // sigma bias
    float* const sTfine = reinterpret_cast<float*>(sb + kOffTfine);
    const float* const sSig = reinterpret_cast<const float*>(sb + kOffSig);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int Dc = P.depth_coarse, Df = P.depth_fine, Dt = Dc + Df;
    const int Tc = K.Tc, Tf = K.Tf;
    const uint64_t seed = P.seed_ptr ? (P.seed + __ldg(reinterpret_cast<const unsigned long long*>(P.seed_ptr))) : P.seed;

    // this CTA's contiguous chunk of groups
    const int g_begin = (int)((K.total_groups * blockIdx.x) / gridDim.x);
    const int n_groups = (int)((K.total_groups * (blockIdx.x + 1)) / gridDim.x) - g_begin;

    // ---- one-time setup
    if (tid == 0) {
        init_pipeline_barriers(S);
        mbar_init(S.bar(BAR_FINE + 0), 4); mbar_init(S.bar(BAR_FINE + 1), 4);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    stage_decoder(sb, P.w0, P.b0, P.w1, P.b1, tid);
    __syncthreads();

    // ============================================================================================================ gather warps
    if (warp >= kEWarps) {
        const int gw = warp - kEWarps;
        uint2* const taps = reinterpret_cast<uint2*>(sb + kOffTaps + gw * kTapBytesPerWarp);
        int next_item = gw;                                   // item = tile * 4 + quarter
        auto item = [&](int ti, int q, bool fine, int r, int t) {
            const int row = q * 32 + lane, rs = row / L, j = row & (L - 1);
            const Ray ray = make_ray(K, g_begin + r, rs);
            const int k = t * L + j;
            const bool valid = ray.ok && k < (fine ? Df : Dc);
            float depth = 0.f;
            if (fine) {
                mbar_wait_sleep(S.bar(BAR_FINE + (r & 1)), (uint32_t)((r >> 1) & 1), 40u);
                if (valid) depth = sTfine[(r & 1) * kTfineFloats + rs * Df + k];
            } else if (valid) {
                depth = coarse_depth(K, seed, ray.gr, k);
            }
            setup_taps(taps, lane, ray.ox + depth * ray.dx, ray.oy + depth * ray.dy, ray.oz + depth * ray.dz, valid, ray.img4, P.PH, P.PW,
                       K.scale);
            fill_buffer(S, P.planes, taps, ti, q * 32, lane);
        };
        auto tile = [&](int ti, bool fine, int r, int t) {
            while (next_item < ti * 4 + 4) {
                item(ti, next_item - ti * 4, fine, r, t);
                next_item += kGWarps;
            }
        };
        TileIter it(n_groups, Tc, Tf);
        for (int i = 0; it.next(); ++i) tile(i, it.kind == 1, it.group(), it.t);
    }
    // ============================================================================================================ epilogue warps
    else {
        const int eset = warp >> 2, q = warp & 3;
        const int row = q * 32 + lane, rs = row / L, j = row & (L - 1), rw = lane / L;
        using Seg = RaySeg<L>;
        float* const es = reinterpret_cast<float*>(sb + kOffEscr) + Seg::area(warp) * kEscrFloats;
        Seg seg(es, warp, lane);
        constexpr int NB = 8 * L;                                   // u-buckets per ray (8 per lane)
        const int strD = Dt + 2;
        float* const s_sd = es + rw * strD;                         // sorted depths
        float* const s_sg = es + Seg::kRays * strD + rw * strD;
        float* const s_wb = es + 2 * Seg::kRays * strD + rw * strD;
        int* const s_ub = reinterpret_cast<int*>(es) + rw * 2 * NB; // [NB] count | prefix << 8, then [NB] member indices (4 bytes)
        float* const s_tc = es + Seg::kTcOff + rw * Dc;
        float* const s_tf = es + Seg::kTfOff + rw * Df;
        int* const s_hist = reinterpret_cast<int*>(es + Seg::kHistOff) + rw * (Dc + 1);

        // state of the group in its fine phase (cur) and of the group in its coarse phase (nxt)
        float cur_tc[kMaxT], cur_sc[kMaxT], cur_tf[kMaxT], cur_sf[kMaxT];
        float nxt_tc[kMaxT], nxt_sc[kMaxT], nxt_tf[kMaxT];
        int cur_pk[kMaxT] = {0, 0, 0}, nxt_pk[kMaxT] = {0, 0, 0};     // per fine sample: u-bucket | cdf bin << 16
        long long cur_gr = 0, nxt_gr = 0;
        bool cur_ok = false, nxt_ok = false;
#pragma unroll
        for (int t = 0; t < kMaxT; ++t) { cur_tc[t] = cur_sc[t] = cur_tf[t] = cur_sf[t] = nxt_tc[t] = nxt_sc[t] = nxt_tf[t] = 0.f; }
        float dmin = INFINITY, dmax = -INFINITY;
        int dimg = 0;                                               // depth_minmax pair dmin / dmax fold into (per-image mode)
        // fold this warp's running depth range into pair dimg and restart it: one atomic pair per warp of set 0 (warp-uniform)
        auto flush_range = [&]() {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                dmin = fminf(dmin, __shfl_xor_sync(FULL, dmin, o));
                dmax = fmaxf(dmax, __shfl_xor_sync(FULL, dmax, o));
            }
            if (lane == 0) {       // depths are positive (ray_start > 0): IEEE ordering == signed-int ordering
                int* const mm = reinterpret_cast<int*>(P.depth_minmax) + 2 * dimg;
                if (dmin < INFINITY) atomicMin(mm, __float_as_int(dmin));
                if (dmax > -INFINITY) atomicMax(mm + 1, __float_as_int(dmax));
            }
            dmin = INFINITY; dmax = -INFINITY;
        };

        // ---- decoder of tile ti, layer 1 (frees the A buffer; hidden layer -> shared memory)
        auto epi1 = [&](int ti) { layer1_tile(S, q, eset, lane, ti); };
        // ---- layer 2 of tile ti: raw sigma -> sSig[ti & 1], sigmoid colours -> slot.  The slot's previous group was composited
        // before this runs (the caller orders it after the pending tile's per-ray phases).
        auto epi_l2 = [&](int ti, int slot) {
            float col[2][2][4], sig[2][4];
            layer2_tile(S, q, eset, lane, true, col, sig);
            const int g4 = lane >> 2, c4 = lane & 3;
            uint32_t* const cs = reinterpret_cast<uint32_t*>(sb + kOffCol + slot * 8192);
            const float* const bc = sB1c;
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    const int r = 32 * q + 16 * mt + g4 + 8 * hr;
#pragma unroll
                    for (int nt = 0; nt < 2; ++nt) {
                        const int ch = 16 * eset + 8 * nt + 2 * c4;
                        const float s0 = fminf(colour_sigmoid(col[mt][nt][2 * hr] + bc[ch]), 1.f);
                        const float s1 = fminf(colour_sigmoid(col[mt][nt][2 * hr + 1] + bc[ch + 1]), 1.f);
                        cs[r * 16 + (ch >> 1)] = __float2uint_rn(s0 * 65535.f) | (__float2uint_rn(s1 * 65535.f) << 16);
                    }
                    if (eset == 0 && c4 == 0) reinterpret_cast<float*>(sb + kOffSig)[(ti & 1) * 128 + r] = sig[mt][2 * hr];
                }
            asm volatile("bar.sync %0, 64;" ::"r"(1 + q) : "memory");   // hidden buffer free, sigma published
        };
        auto read_sigma = [&](int tj) -> float { return sSig[(tj & 1) * 128 + row] + sB1s[0]; };

        // ---- coarse weights -> smoothed pdf -> cdf -> inverse-CDF fine depths (renderer.py:209-268) for the group in `nxt`
        auto importance = [&](int r) {
            float w[kMaxT], tm[kMaxT];
            seg.enter();
            march_weights(seg, nxt_tc, nxt_sc, Dc, j, w, tm);
            // max_pool1d(k2,s1,pad1) -> avg_pool1d(k2,s1) -> + 0.01; entries [1:-1] => pdf weights at k = 1 .. Dc-3, + 1e-5
            const int nw = Dc - 3;
            float c[kMaxT], wp[kMaxT], wn[kMaxT];
            float part = 0.f;
            seg.prev(w, 0.f, wp);
            seg.next(w, 0.f, wn);
#pragma unroll
            for (int t = 0; t < kMaxT; ++t) {
                const int k = t * L + j;
                c[t] = (k >= 1 && k <= nw) ? (fmaxf(wp[t], w[t]) + fmaxf(w[t], wn[t])) * 0.5f + 0.01f + 1e-5f : 0.f;
                part += c[t];
            }
            const float total = seg.sum(part);
#pragma unroll
            for (int t = 0; t < kMaxT; ++t) c[t] = c[t] / total;
            seg.template scan<false>(c);                            // c[t] = cdf[k], k = 0 .. nw
            float* const cdf = s_sd;
#pragma unroll
            for (int t = 0; t < kMaxT; ++t) {
                const int k = t * L + j;
                if (k <= nw) cdf[k] = c[t];
                if (k < Dc) s_tc[k] = nxt_tc[t];
            }
            seg.sync();
            float uu[kMaxT];
            int lo[kMaxT], hi[kMaxT];
#pragma unroll
            for (int t = 0; t < kMaxT; ++t) {
                const int jf = t * L + j;
                const bool act = jf < Df && nxt_ok;
                uu[t] = !act ? 0.f : P.u_fine ? __ldg(P.u_fine + nxt_gr * Df + jf) : hash_uniform(seed ^ 0xA5A5A5A5DEADBEEFull, (uint64_t)(nxt_gr * Df + jf));
                lo[t] = 0;
                hi[t] = act ? nw + 1 : 0;                            // searchsorted(cdf, u, right=True): first index with cdf[idx] > u
            }
            const int nit = 32 - __clz(nw + 1);
            for (int it = 0; it < nit; ++it) {                       // the three searches of a lane advance together (independent chains)
#pragma unroll
                for (int t = 0; t < kMaxT; ++t)
                    if (lo[t] < hi[t]) { const int mid = (lo[t] + hi[t]) >> 1; if (cdf[mid] <= uu[t]) lo[t] = mid + 1; else hi[t] = mid; }
            }
#pragma unroll
            for (int t = 0; t < kMaxT; ++t) {
                const int jf = t * L + j;
                float tf = 0.f;
                int below = 0;
                if (jf < Df && nxt_ok) {
                    below = max(lo[t] - 1, 0);
                    const int above = min(lo[t], nw);
                    const float cb = cdf[below], ca = cdf[above];
                    const float bb = 0.5f * (s_tc[below] + s_tc[below + 1]), ba = 0.5f * (s_tc[above] + s_tc[above + 1]);
                    float denom = ca - cb;
                    if (denom < 1e-5f) denom = 1.f;
                    tf = bb + (uu[t] - cb) / denom * (ba - bb);
                }
                nxt_tf[t] = tf;
                nxt_pk[t] = min(NB - 1, (int)(uu[t] * (float)NB)) | (below << 16);
                if (eset == 0 && jf < Df) sTfine[(r & 1) * kTfineFloats + rs * Df + jf] = tf;
            }
            __syncwarp();
            if (eset == 0 && lane == 0) mbar_arrive(S.bar(BAR_FINE + (r & 1)));
        };

        // ---- final weights + colour composite of group r (state in cur_*).  use_fine: merge coarse + fine; else coarse only.
        auto composite = [&](int r, bool use_fine) {
            const float (&tc)[kMaxT] = cur_tc;
            const float (&sc)[kMaxT] = cur_sc;
            const long long gr = cur_gr;
            const bool ok = cur_ok;
            const int cnt = use_fine ? Dt : Dc;
            float coef_c[kMaxT], coef_f[kMaxT];
            float wsum, dacc;
            float d_first, d_last;
            // the ray's `cnt` depth-sorted samples (depths d, final weights w, interval midpoints tm): export them, sum the weights
            // and weight x midpoint over the ray, take the first depth
            auto ray_sums = [&](const auto& d, const auto& w, const auto& tm) {
                constexpr int NT = sizeof(d) / sizeof(d[0]);
                if constexpr (kExport) {
                    if (ok && eset == 0) {                           // both warp sets hold the ray; one writes
                        float* const out = K.samples + gr * (2 * cnt - 1);
#pragma unroll
                        for (int t = 0; t < NT; ++t) {
                            const int p = t * L + j;
                            if (p < cnt) out[p] = d[t];
                            if (p < cnt - 1) out[cnt + p] = w[t];
                        }
                    }
                }
                float ws = 0.f, da = 0.f;
#pragma unroll
                for (int t = 0; t < NT; ++t) { ws += w[t]; da += w[t] * tm[t]; }
                wsum = seg.sum(ws);
                dacc = seg.sum(da);
                d_first = seg.lead(d[0]);                            // read on j == 0 only
            };
            seg.enter();
            if (use_fine) {
                // stable sort-merge of coarse (sorted) + fine depths by rank (torch.sort of the concatenation, renderer.py:164-182)
#pragma unroll
                for (int t = 0; t < kMaxT; ++t) {
                    const int k = t * L + j;
                    if (k < Dc) s_tc[k] = tc[t];
                    if (k < Df) s_tf[k] = cur_tf[t];
                    if (k <= Dc) s_hist[k] = 0;
                }
                if (j == 0 && L * kMaxT <= Dc) s_hist[Dc] = 0;
                seg.sync();
                // zero the u-bucket tables (they alias the sorted arrays, which are written after the ranks are known)
                for (int i = j; i < 2 * NB; i += L) s_ub[i] = 0;
                seg.sync();
                // Rank of a fine sample among the fine ones.  Fine depths are the inverse CDF of iid uniforms u, a monotone map, so the
                // order of the depths is the order of the u's: bucket the samples by u (NB uniform buckets, ~0.4 samples each), take
                // the bucket prefix count and order the few members of a bucket by (depth, index).  The number of coarse samples <= v
                // follows from the CDF bin the sample was drawn from (its depth lies between the midpoints around that bin).
                int pos_f[kMaxT], pos_c[kMaxT], cntc[kMaxT];
                bool overflow = false;
#pragma unroll
                for (int t = 0; t < kMaxT; ++t) {
                    const int jf = t * L + j;
                    cntc[t] = 0;
                    if (jf < Df) {
                        const float v = cur_tf[t];
                        const int key = cur_pk[t] & 0xffff, below = cur_pk[t] >> 16;
                        const int slot = atomicAdd(&s_ub[key], 1);
                        if (slot < 4) atomicOr(&s_ub[NB + key], jf << (8 * slot));
                        int c = below + 1 + (s_tc[below + 1] <= v ? 1 : 0);
                        if (c == below + 2 && c < Dc && s_tc[c] <= v) ++c;
                        if (!(s_tc[c - 1] <= v && (c == Dc || s_tc[c] > v))) {       // never taken unless the bracket argument fails: search
                            int lo = 0, hi = Dc;
                            while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_tc[mid] <= v) lo = mid + 1; else hi = mid; }
                            c = lo;
                        }
                        cntc[t] = c;
                        atomicAdd(&s_hist[c], 1);
                    }
                }
                seg.sync();
                {   // exclusive prefix over the buckets: lane j owns buckets 8j .. 8j+7; count and prefix share a word
                    int cn[8], run = 0;
#pragma unroll
                    for (int i = 0; i < 8; ++i) { cn[i] = s_ub[8 * j + i]; run += cn[i]; }
                    int pre = seg.prefix(run) - run;
#pragma unroll
                    for (int i = 0; i < 8; ++i) { s_ub[8 * j + i] = cn[i] | (pre << 8); pre += cn[i]; }
                }
                seg.sync();
#pragma unroll
                for (int t = 0; t < kMaxT; ++t) {
                    const int jf = t * L + j;
                    pos_f[t] = 0;
                    if (jf < Df) {
                        const float v = cur_tf[t];
                        const int key = cur_pk[t] & 0xffff;
                        const int word = s_ub[key], cn = word & 255;
                        const int mem = s_ub[NB + key];
                        int within = 0;
                        if (cn > 4) overflow = true;
                        else {
#pragma unroll
                            for (int m = 0; m < 4; ++m) {
                                const int idx = (mem >> (8 * m)) & 255;
                                if (m < cn && idx != jf) { const float x = s_tf[idx]; within += (x < v || (x == v && idx < jf)) ? 1 : 0; }
                            }
                        }
                        pos_f[t] = cntc[t] + (word >> 8) + within;
                    }
                }
                if (seg.any(overflow)) {                             // a crowded bucket (degenerate u's): full O(Df^2) rank count
#pragma unroll
                    for (int t = 0; t < kMaxT; ++t) {
                        const int jf = t * L + j;
                        if (jf < Df) {
                            const float v = cur_tf[t];
                            int cntf = 0;
                            for (int i = 0; i < Df; ++i) { const float x = s_tf[i]; cntf += (x < v || (x == v && i < jf)) ? 1 : 0; }
                            pos_f[t] = cntc[t] + cntf;
                        }
                    }
                }
                seg.sync();
                // coarse sample a lands after every fine sample with fewer than a+1 coarse samples <= it: a + #{fine: cnt_c <= a}
                float hc[kMaxT];
#pragma unroll
                for (int t = 0; t < kMaxT; ++t) { const int k = t * L + j; hc[t] = k < Dc ? (float)s_hist[k] : 0.f; }
                seg.template scan<false>(hc);
#pragma unroll
                for (int t = 0; t < kMaxT; ++t) {
                    const int k = t * L + j;
                    pos_c[t] = k + (int)hc[t];
                    if (k < Dc) { s_sd[pos_c[t]] = tc[t]; s_sg[pos_c[t]] = sc[t]; }
                    if (k < Df) { s_sd[pos_f[t]] = cur_tf[t]; s_sg[pos_f[t]] = cur_sf[t]; }
                }
                seg.sync();
                float d6[2 * kMaxT], s6[2 * kMaxT], w6[2 * kMaxT], tm6[2 * kMaxT];
#pragma unroll
                for (int t = 0; t < 2 * kMaxT; ++t) {
                    const int p = t * L + j;
                    d6[t] = p < cnt ? s_sd[p] : 0.f;
                    s6[t] = p < cnt ? s_sg[p] : 0.f;
                }
                march_weights(seg, d6, s6, cnt, j, w6, tm6);
                ray_sums(d6, w6, tm6);
                if (j == 0) s_wb[0] = 0.f;
#pragma unroll
                for (int t = 0; t < 2 * kMaxT; ++t) {
                    const int p = t * L + j;
                    if (p < cnt) s_wb[p + 1] = w6[t];
                }
                seg.sync();
                d_last = s_sd[cnt - 1];
#pragma unroll
                for (int t = 0; t < kMaxT; ++t) {
                    const int k = t * L + j;
                    coef_c[t] = k < Dc ? 0.5f * (s_wb[pos_c[t]] + s_wb[pos_c[t] + 1]) : 0.f;
                    coef_f[t] = k < Df ? 0.5f * (s_wb[pos_f[t]] + s_wb[pos_f[t] + 1]) : 0.f;
                }
            } else {
                float w3[kMaxT], tm3[kMaxT], wp[kMaxT];
                march_weights(seg, tc, sc, cnt, j, w3, tm3);
                ray_sums(tc, w3, tm3);
                seg.prev(w3, 0.f, wp);
#pragma unroll
                for (int t = 0; t < kMaxT; ++t) {
                    const int k = t * L + j;
                    coef_c[t] = k < Dc ? 0.5f * ((k > 0 ? wp[t] : 0.f) + w3[t]) : 0.f;
                    coef_f[t] = 0.f;
                }
                if (j == 0) s_wb[0] = 0.f;                          // keep the scratch race-free across phases
#pragma unroll
                for (int t = 0; t < kMaxT; ++t) { const int k = t * L + j; if (k < Dc) s_sd[k] = tc[t]; }
                seg.sync();
                d_last = s_sd[Dc - 1];
            }
            // colours: acc[c] += coef * sigmoid(logit + b1) over this thread's rows, channels 16*eset .. +15 (sigmoid * 1.002 - 0.001,
            // triplane_next3d.py:369-370, is affine: applied once to the sum)
            float acc[16];
#pragma unroll
            for (int c = 0; c < 16; ++c) acc[c] = 0.f;
            auto add_tile = [&](int slot, float coef) {
                const uint4* src = reinterpret_cast<const uint4*>(sb + kOffCol + slot * 8192 + row * 64 + 32 * eset);
                const uint4 u0 = src[0], u1 = src[1];
                const uint32_t v[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    acc[2 * c] = fmaf(coef, (float)(v[c] & 0xffffu) * (1.f / 65535.f), acc[2 * c]);
                    acc[2 * c + 1] = fmaf(coef, (float)(v[c] >> 16) * (1.f / 65535.f), acc[2 * c + 1]);
                }
            };
#pragma unroll
            for (int t = 0; t < kMaxT; ++t)
                if (t < Tc) add_tile((r & 1) * 3 + t, coef_c[t]);
            if (use_fine) {
#pragma unroll
                for (int t = 0; t < kMaxT; ++t)
                    if (t < Tf) add_tile(6 + t, coef_f[t]);
            }
            seg.reduce16(acc);                                      // lane j < 16 now holds channel j of the ray
            if (ok && j < 16) {
                float v = fmaf(acc[0], 1.002f, -0.001f * wsum);     // sum_k coef_k (1.002 sigmoid_k - 0.001), sum_k coef_k = wsum
                if (P.white_back) v = v + 1.f - wsum;
                P.rgb[gr * kFeat + 16 * eset + j] = v * 2.f - 1.f;
            }
            if (P.depth_range_per_image && eset == 0) {              // a group's rays all belong to image (g_begin + r) / gpi
                const int n = (g_begin + r) / K.gpi;
                if (n != dimg) { flush_range(); dimg = n; }
            }
            if (ok && eset == 0 && j == 0) {
                float depth = dacc / wsum;
                if (isnan(depth)) depth = INFINITY;                  // nan_to_num(nan=inf); the clamp kernel finishes the job
                P.depth[gr] = depth;
                P.wsum[gr] = wsum;
                dmin = fminf(dmin, d_first);
                dmax = fmaxf(dmax, d_last);
            }
        };

        // ---- sigma of tile (kind, r, t) arrived: store it; the last tile of a pass triggers the per-ray phases
        int pend_kind = -1, pend_r = 0, pend_t = 0, pend_i = 0;      // kind: 0 coarse, 1 fine
        auto epi2 = [&]() {
            const float sg = read_sigma(pend_i);
            bool do_composite = false, shift = false;
            if (pend_kind == 0) {
#pragma unroll
                for (int t = 0; t < kMaxT; ++t) if (t == pend_t) nxt_sc[t] = sg;
                if (pend_t == Tc - 1) {
                    // depths + ray of the coarse group
                    const RayId id = ray_of(K, g_begin + pend_r, rs);
                    nxt_ok = id.ok; nxt_gr = id.gr;
#pragma unroll
                    for (int t = 0; t < kMaxT; ++t) { const int k = t * L + j; nxt_tc[t] = (id.ok && k < Dc) ? coarse_depth(K, seed, id.gr, k) : 0.f; }
                    if (Tf > 0) {
                        importance(pend_r);
                        shift = pend_r == 0;                        // the first group moves to its fine phase right away
                    } else {
                        shift = true;                               // coarse-only rendering: composite straight from the coarse pass
                        do_composite = true;
                    }
                }
            } else {
#pragma unroll
                for (int t = 0; t < kMaxT; ++t) if (t == pend_t) cur_sf[t] = sg;
                do_composite = pend_t == Tf - 1;
            }
            if (shift) {
#pragma unroll
                for (int t = 0; t < kMaxT; ++t) { cur_tc[t] = nxt_tc[t]; cur_sc[t] = nxt_sc[t]; cur_tf[t] = nxt_tf[t]; cur_pk[t] = nxt_pk[t]; }
                cur_gr = nxt_gr; cur_ok = nxt_ok;
            }
            if (do_composite) {
                composite(pend_r, pend_kind == 1);
                if (pend_kind == 1) {                               // the next group (already importance-sampled) enters its fine phase
#pragma unroll
                    for (int t = 0; t < kMaxT; ++t) { cur_tc[t] = nxt_tc[t]; cur_sc[t] = nxt_sc[t]; cur_tf[t] = nxt_tf[t]; cur_pk[t] = nxt_pk[t]; }
                    cur_gr = nxt_gr; cur_ok = nxt_ok;
                }
            }
        };

        TileIter it(n_groups, Tc, Tf);
        for (int i = 0;; ++i) {
            const bool has = it.next();
            // a fine tile directly behind the coarse tiles of its own group (single-group CTA): its depths come out of the pending
            // coarse epilogue, which therefore cannot be deferred behind this tile's layer-1 epilogue
            const bool early = has && it.kind == 1 && pend_kind == 0 && pend_r == it.group();
            if (has && !early) epi1(i);
            if (pend_kind >= 0) epi2();
            if (!has) break;
            if (early) epi1(i);
            // colour slot: coarse tiles of even / odd groups in 0-2 / 3-5, fine tiles in 6-8; written after the pending tile's
            // per-ray phases, which composite the group that used the slot before
            epi_l2(i, it.kind == 0 ? (it.group() & 1) * 3 + it.t : 6 + it.t);
            pend_kind = it.kind; pend_r = it.group(); pend_t = it.t; pend_i = i;
        }

        // depth range (ray_marcher.py:54): batch-global into pair 0, or per image into pair dimg (the last image this warp composited)
        if (eset == 0 && P.depth_minmax) flush_range();
    }

}

// ---------------------------------------------------------------------------------------------------------------- run_model
// Decoder on arbitrary points (renderer.run_model, renderer.py:149-155; TriPlaneGenerator.sample, triplane_next3d.py:232-276) with the
// same gather / tensor-core epilogue roles as the renderer, minus the per-ray phases.  Tile = 128 consecutive points.  In grid mode
// (coords == nullptr) the points are the voxel centres of create_samples (gen_samples_next3d.py:80-102), generated in the kernel
// with the script's own float32 operations, and the flip + border trim of gen_samples_next3d.py:226-238 is applied on the way
// out: voxels in the trimmed border get pad_value and are never decoded.
struct PointsK {
    const float* planes;
    int N, PH, PW;
    const float* coords;         // [N, Pn, 3] or nullptr (grid mode, N = 1)
    long long Pn, total;         // points per image, N * Pn
    float scale;
    const float* w0; const float* b0; const float* w1; const float* b1;
    float* sigma;                // [N, Pn]  (grid mode: [R, R, R] already flipped + trimmed)
    float* rgb;                  // [N, Pn, 32] or nullptr
    int grid_n, pad;             // grid mode: voxels per side, trimmed border width
    float voxel_size, org0, org1, org2, pad_value;
    long long head;              // grid mode: flat index of the first point
};

// voxel centre of flat index idx, bit-identical to the reference's float32 expression chain (float, not floor, division)
__device__ __forceinline__ void grid_point(const PointsK& K, long long idx, float& x, float& y, float& z) {
    const float fn = (float)K.grid_n;
    const float fi = (float)idx;                                   // int64 -> float32, round to nearest (indices above 2^24 lose bits)
    const float s2 = (float)(idx % K.grid_n);
    const float q1 = __fdiv_rn(fi, fn);
    const float s1 = fmodf(q1, fn);
    const float s0 = fmodf(__fdiv_rn(q1, fn), fn);
    x = __fadd_rn(__fmul_rn(s0, K.voxel_size), K.org2);
    y = __fadd_rn(__fmul_rn(s1, K.voxel_size), K.org1);
    z = __fadd_rn(__fmul_rn(s2, K.voxel_size), K.org0);
}
// destination of flat index idx after flip(dims=[0]) and whether it lies in the trimmed border
__device__ __forceinline__ long long grid_dest(const PointsK& K, long long idx, bool& border) {
    const long long n = K.grid_n;
    const long long a = idx / (n * n), rem = idx - a * n * n;
    const long long b = rem / n, c = rem - b * n;
    const long long fa = n - 1 - a;
    border = fa < K.pad || fa >= n - K.pad || b < K.pad || b >= n - K.pad || c < K.pad || c >= n - K.pad;
    return (fa * n + b) * n + c;
}

template <bool RGB>
__global__ void __launch_bounds__(kThreads, 1) points_fused_kernel(const __grid_constant__ PointsK K) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    Smem S;
    S.base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* const sb = S.base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool grid = K.coords == nullptr;

    const long long n_tiles_all = (K.total + 127) / 128;
    // tiles are dealt round-robin: the skipped border tiles of a trimmed grid are spread evenly over the CTAs
    const long long t_begin = blockIdx.x, t_end = n_tiles_all, t_step = gridDim.x;
    // a tile of the voxel grid is skipped when every one of its points falls into the trimmed border
    auto tile_skipped = [&](long long tile) -> bool {
        if (!grid || K.pad <= 0) return false;
        const long long first = K.head + tile * 128, last = min(K.head + K.total, first + 128) - 1;
        const long long n = K.grid_n, r0 = first / n, r1 = last / n;           // rows (a, b) touched: at most r0 .. r1
        for (long long r = r0; r <= r1; ++r) {
            const long long a = r / n, b = r - a * n, fa = n - 1 - a;
            if (!(fa < K.pad || fa >= n - K.pad || b < K.pad || b >= n - K.pad)) return false;
        }
        return true;
    };

    if (tid == 0) {
        init_pipeline_barriers(S);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    stage_decoder(sb, K.w0, K.b0, K.w1, K.b1, tid);
    __syncthreads();

    if (warp >= kEWarps) {                                         // ---- gather warps
        const int gw = warp - kEWarps;
        uint2* const taps = reinterpret_cast<uint2*>(sb + kOffTaps + gw * kTapBytesPerWarp);
        int next_item = gw, i = 0;
        for (long long tile = t_begin; tile < t_end; tile += t_step) {
            if (tile_skipped(tile)) continue;
            while (next_item < i * 4 + 4) {
                const int q = next_item - i * 4;
                const long long g = tile * 128 + q * 32 + lane;
                bool valid = g < K.total;
                float px = 0.f, py = 0.f, pz = 0.f;
                uint32_t img = 0;
                if (valid) {
                    if (grid) {
                        bool border;
                        grid_dest(K, K.head + g, border);
                        valid = !border;
                        grid_point(K, K.head + g, px, py, pz);
                    } else {
                        const float* c = K.coords + g * 3;
                        px = __ldg(c); py = __ldg(c + 1); pz = __ldg(c + 2);
                        img = (uint32_t)(g / K.Pn) * (uint32_t)(3 * K.PH * K.PW * 128);
                    }
                }
                setup_taps(taps, lane, px, py, pz, valid, img, K.PH, K.PW, K.scale);
                fill_buffer(S, K.planes, taps, i, q * 32, lane);
                next_item += kGWarps;
            }
            ++i;
        }
    } else {                                                       // ---- epilogue warps
        const int eset = warp >> 2, q = warp & 3;
        const float* const sB1c = reinterpret_cast<const float*>(sb + kOffBias) + 64;
        const float sB1s = reinterpret_cast<const float*>(sb + kOffBias)[96];
        const int g4 = lane >> 2, c4 = lane & 3;
        int i = 0;
        for (long long tile = t_begin; tile < t_end; tile += t_step) {
            if (tile_skipped(tile)) {                              // whole tile in the trimmed border: only the pad value is written
                const long long g = tile * 128 + q * 32 + lane;
                if (eset == 0 && g < K.total) { bool border; K.sigma[grid_dest(K, K.head + g, border)] = K.pad_value; }
                continue;
            }
            layer1_tile(S, q, eset, lane, i);
            float col[2][2][4], sig[2][4];
            layer2_tile(S, q, eset, lane, RGB, col, sig);
            asm volatile("bar.sync %0, 64;" ::"r"(1 + q) : "memory");   // hidden buffer free for the next tile
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    const long long g = tile * 128 + 32 * q + 16 * mt + g4 + 8 * hr;
                    if (g >= K.total) continue;
                    if (RGB) {
#pragma unroll
                        for (int nt = 0; nt < 2; ++nt) {
                            const int ch = 16 * eset + 8 * nt + 2 * c4;
                            float2 o;                               // sigmoid(x) * 1.002 - 0.001 (triplane_next3d.py:369-370)
                            o.x = fmaf(colour_sigmoid(col[mt][nt][2 * hr] + sB1c[ch]), 1.002f, -0.001f);
                            o.y = fmaf(colour_sigmoid(col[mt][nt][2 * hr + 1] + sB1c[ch + 1]), 1.002f, -0.001f);
                            *reinterpret_cast<float2*>(K.rgb + g * kFeat + ch) = o;
                        }
                    }
                    if (eset == 0 && c4 == 0) {
                        const float sg = sig[mt][2 * hr] + sB1s;
                        if (grid) {
                            bool border;
                            const long long d = grid_dest(K, K.head + g, border);
                            K.sigma[d] = border ? K.pad_value : sg;
                        } else {
                            K.sigma[g] = sg;
                        }
                    }
                }
            ++i;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------- normals
// n = -grad_x sigma_raw at every sample the renderer composited, composited with the renderer's final weights
// (renderer.py:271-355 normal_forward, ray_marcher.py:32-33, 61-64).  Input: the sorted depths and final interval weights that
// render_fused_kernel<L, true> exported per ray.  Per sample, from ONE fetch of its 12 bilinear taps:
//   f = plane-mean feature and J_a = d f / d x_a (a = x, y, z; the bilinear-derivative weights of the same tap fractions),
//   sigma' = sigmoid(W0 f + b0) (softplus' = sigmoid),  d sigma / d x_a = sum_k sigma'_k W1[0, k] (W0 J_a)_k,
// evaluated in reverse mode: g = W0^T (sigma' * W1[0, :]) = d sigma / d f on the tensor cores, then three 32-long dot products
// g . J_a (DESIGN.md section 3.2a).
// One warp = one ray at a time, 16 samples per chunk (tile row = sample); every product runs on mma.sync m16n8k16, bf16x3 with fp32
// accumulation, like the renderer's decoder.  The layer-1 accumulator fragments feed the second product directly as its A operand.
struct NormalsK {
    N3DRender p;
    int D;                       // samples per ray in `samples`: Dc + Df, or Dc when coarse-only
    float scale;                 // 2 / box_warp
    long long rays;              // N * res * res
    const float* samples;        // [rays][2D - 1]: D sorted depths, then D - 1 final weights
    float* normal;               // [rays][3]
};

constexpr int kNWarps = 8, kNThreads = kNWarps * 32;
constexpr int kNRows = 16;                                      // samples per chunk
constexpr int kNFrags = 64;                                     // B fragments per lane: 32 of W0^T (layer 1), then 32 of W0 (layer 1 transposed)
constexpr int kNOffB0 = kNFrags * 32 * 8;                       // [kNFrags][32 lanes] (hi, lo) words, then b0 [64] | W1[0, :] [64]
constexpr int kNJStride = 100;                                  // floats per row of the fp32 J tile ([3][32] + pad)
constexpr int kNOffWarp = kNOffB0 + 2 * kHidden * 4;
// per warp: f tile hi | lo ([16] x 64-byte SWIZZLE_64B rows), then the J tile [16][kNJStride] fp32
constexpr int kNJBytes = kNRows * kNJStride * 4;
constexpr int kNWarpBytes = 2 * kNRows * 64 + kNJBytes;
constexpr int kNSmemBytes = kNOffWarp + kNWarps * kNWarpBytes;  // 84480: two CTAs per SM

// Layer 1 of the 16 rows of a bf16 (hi, lo) SWIZZLE_64B tile: acc[nt] = rows x hidden units 8 nt .. 8 nt + 7 (m16n8 fragments).
__device__ __forceinline__ void normals_layer1(const uint8_t* th, const uint8_t* tl, const uint2* frag, int lane, float (&acc)[8][4]) {
    const int g = lane >> 2, c = lane & 3;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
#pragma unroll
    for (int ks = 0; ks < kFeat / 16; ++ks) {
        uint32_t ah[4], al[4];
        ah[0] = lds32(th + sw64_off(g, ks * 32 + 4 * c)); ah[1] = lds32(th + sw64_off(g + 8, ks * 32 + 4 * c));
        ah[2] = lds32(th + sw64_off(g, ks * 32 + 16 + 4 * c)); ah[3] = lds32(th + sw64_off(g + 8, ks * 32 + 16 + 4 * c));
        al[0] = lds32(tl + sw64_off(g, ks * 32 + 4 * c)); al[1] = lds32(tl + sw64_off(g + 8, ks * 32 + 4 * c));
        al[2] = lds32(tl + sw64_off(g, ks * 32 + 16 + 4 * c)); al[3] = lds32(tl + sw64_off(g + 8, ks * 32 + 16 + 4 * c));
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const uint2 b0 = frag[((ks * 8 + nt) * 2) * 32 + lane], b1 = frag[((ks * 8 + nt) * 2 + 1) * 32 + lane];
            mma_bf16_16816(acc[nt], ah, b0.x, b1.x);
            mma_bf16_16816(acc[nt], ah, b0.y, b1.y);
            mma_bf16_16816(acc[nt], al, b0.x, b1.x);
        }
    }
}

__device__ __forceinline__ void store_split_row(uint8_t* th, uint8_t* tl, int row, int c, const float (&v)[8]) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) split_bf16x2(v[2 * q], v[2 * q + 1], h[q], l[q]);
    const uint32_t off = sw64_off(row, c * 16);
    *reinterpret_cast<uint4*>(th + off) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(tl + off) = make_uint4(l[0], l[1], l[2], l[3]);
}

__global__ void __launch_bounds__(kNThreads, 2) normals_fused_kernel(const __grid_constant__ NormalsK K) {
    extern __shared__ __align__(16) uint8_t nsm[];
    const N3DRender& P = K.p;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint2* const frag = reinterpret_cast<const uint2*>(nsm);
    const float* const sB0 = reinterpret_cast<const float*>(nsm + kNOffB0);
    const float* const sW1 = sB0 + kHidden;

    // ---- B fragments (mma.m16n8k16: b0 = B[2c, 2c+1][g], b1 = B[2c+8, 2c+9][g]) split into bf16 (hi, lo), one (hi, lo) pair per lane
    for (int i = tid; i < kNFrags * 32; i += kNThreads) {
        const int f = i >> 5, g = (i >> 2) & 7, c = i & 3;
        float v0, v1;
        if (f < 32) {            // B[k = feature][n = hidden] = W0[n][k];  f = (ks * 8 + nt) * 2 + reg
            const int ks = f >> 4, nt = (f >> 1) & 7, k0 = 16 * ks + 8 * (f & 1) + 2 * c;
            v0 = __ldg(P.w0 + (8 * nt + g) * kFeat + k0);
            v1 = __ldg(P.w0 + (8 * nt + g) * kFeat + k0 + 1);
        } else {                 // B[k = hidden][n = feature] = W0[k][n];  f - 32 = (ks * 4 + nt) * 2 + reg
            const int e = f - 32, ks = e >> 3, nt = (e >> 1) & 3, k0 = 16 * ks + 8 * (e & 1) + 2 * c;
            v0 = __ldg(P.w0 + k0 * kFeat + 8 * nt + g);
            v1 = __ldg(P.w0 + (k0 + 1) * kFeat + 8 * nt + g);
        }
        uint32_t h, l;
        split_bf16x2(v0, v1, h, l);
        reinterpret_cast<uint2*>(nsm)[i] = make_uint2(h, l);
    }
    for (int i = tid; i < kHidden; i += kNThreads) {
        reinterpret_cast<float*>(nsm + kNOffB0)[i] = __ldg(P.b0 + i);
        reinterpret_cast<float*>(nsm + kNOffB0)[kHidden + i] = __ldg(P.w1 + i);       // sigma row of W1
    }
    __syncthreads();

    uint8_t* const fh = nsm + kNOffWarp + warp * kNWarpBytes;
    uint8_t* const fl = fh + kNRows * 64;
    float* const jt = reinterpret_cast<float*>(fh + 2 * kNRows * 64);      // J tile
    const char* const planes = reinterpret_cast<const char*>(P.planes);
    const int g = lane >> 2, c = lane & 3;               // fetch: sample g of a step, channel octet c; mma: fragment row g, column pair c
    const int D = K.D, M = P.res * P.res;
    const long long warps = (long long)gridDim.x * kNWarps;
    for (long long gr = (long long)blockIdx.x * kNWarps + warp; gr < K.rays; gr += warps) {
        const int n = (int)(gr / M), m = (int)(gr - (long long)n * M);
        float o[3], d[3];
        camera_ray(P, n, m / P.res, m % P.res, o, d);
        const uint32_t img4 = (uint32_t)(n / P.views) * (uint32_t)(3 * P.PH * P.PW * 128);
        const float* const ts = K.samples + gr * (2 * D - 1);
        const float* const wts = ts + D;
        float nacc[3] = {0.f, 0.f, 0.f}, wsum = 0.f;
        for (int i0 = 0; i0 < D; i0 += kNRows) {
            // ---- fetch: f and J_x, J_y, J_z of samples i0 .. i0 + 15 from one read of the 12 taps; 8 samples x 4 channel octets per
            // step, so lane (g, c) fetches rows g and g + 8 -- the two rows its mma fragments hold
#pragma unroll 1
            for (int step = 0; step < 2; ++step) {
                const int row = step * 8 + g, i = i0 + row;
                const bool valid = i < D;
                const float t = valid ? __ldg(ts + i) : 0.f;
                const float x = K.scale * (o[0] + t * d[0]), y = K.scale * (o[1] + t * d[1]), z = K.scale * (o[2] + t * d[2]);
                float fv[8], jv[3][8];
#pragma unroll
                for (int ch = 0; ch < 8; ++ch) { fv[ch] = 0.f; jv[0][ch] = 0.f; jv[1][ch] = 0.f; jv[2][ch] = 0.f; }
#pragma unroll 1
                for (int pl = 0; pl < 3; ++pl) {                  // one plane's four taps in flight: keeps the 32 accumulators in registers
                    const PlaneTaps tp = plane_taps(pl, x, y, z, valid, img4, P.PH, P.PW, K.scale);
                    float v[4][8], da[8], db[8];
#pragma unroll
                    for (int cc = 0; cc < 4; ++cc) ldg_nc_256(reinterpret_cast<const float*>(planes + tp.off[cc] + c * 32), v[cc]);
#pragma unroll
                    for (int ch = 0; ch < 8; ++ch) {
                        da[ch] = 0.f; db[ch] = 0.f;
#pragma unroll
                        for (int cc = 0; cc < 4; ++cc) {
                            fv[ch] = fmaf(tp.w[cc], v[cc][ch], fv[ch]);
                            da[ch] = fmaf(tp.wa[cc], v[cc][ch], da[ch]);
                            db[ch] = fmaf(tp.wb[cc], v[cc][ch], db[ch]);
                        }
                        // plane 0 <- (x, y), 1 <- (x, z), 2 <- (z, y)
                        jv[0][ch] += pl != 2 ? da[ch] : 0.f;
                        jv[1][ch] += pl != 1 ? db[ch] : 0.f;
                        jv[2][ch] += pl == 1 ? db[ch] : (pl == 2 ? da[ch] : 0.f);
                    }
                }
                store_split_row(fh, fl, row, c, fv);
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    float* const dst = jt + row * kNJStride + a * 32 + c * 8;
                    *reinterpret_cast<float4*>(dst) = make_float4(jv[a][0], jv[a][1], jv[a][2], jv[a][3]);
                    *reinterpret_cast<float4*>(dst + 4) = make_float4(jv[a][4], jv[a][5], jv[a][6], jv[a][7]);
                }
            }
            __syncwarp();
            // ---- u = sigmoid(W0 f + b0) * W1[0, :] for the 16 rows
            float u[8][4];
            normals_layer1(fh, fl, frag, lane, u);
#pragma unroll
            for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int k = 8 * nt + 2 * c + (e & 1);
                    u[nt][e] = sigmoid_fast(u[nt][e] + sB0[k]) * sW1[k];
                }
            float gs[2][3];                                  // d sigma / d x_a of rows g (hr 0) and g + 8 (hr 1), partial over this lane's columns
            // g [16 x 32] = u W0: the accumulator fragments of hidden units 16 ks .. 16 ks + 15 are the A fragment of k-step ks
            float gacc[4][4];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) gacc[nt][e] = 0.f;
#pragma unroll
            for (int ks = 0; ks < kHidden / 16; ++ks) {
                uint32_t ah[4], al[4];
                split_bf16x2(u[2 * ks][0], u[2 * ks][1], ah[0], al[0]);
                split_bf16x2(u[2 * ks][2], u[2 * ks][3], ah[1], al[1]);
                split_bf16x2(u[2 * ks + 1][0], u[2 * ks + 1][1], ah[2], al[2]);
                split_bf16x2(u[2 * ks + 1][2], u[2 * ks + 1][3], ah[3], al[3]);
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    const uint2 b0 = frag[(32 + (ks * 4 + nt) * 2) * 32 + lane], b1 = frag[(32 + (ks * 4 + nt) * 2 + 1) * 32 + lane];
                    mma_bf16_16816(gacc[nt], ah, b0.x, b1.x);
                    mma_bf16_16816(gacc[nt], ah, b0.y, b1.y);
                    mma_bf16_16816(gacc[nt], al, b0.x, b1.x);
                }
            }
            // g . J_a over this lane's 8 features of rows g and g + 8
#pragma unroll
            for (int hr = 0; hr < 2; ++hr)
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    const float* const jr = jt + (g + 8 * hr) * kNJStride + a * 32 + 2 * c;
                    float s = 0.f;
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) {
                        const float2 j2 = *reinterpret_cast<const float2*>(jr + 8 * nt);
                        s = fmaf(gacc[nt][2 * hr], j2.x, fmaf(gacc[nt][2 * hr + 1], j2.y, s));
                    }
                    gs[hr][a] = s;
                }
#pragma unroll
            for (int hr = 0; hr < 2; ++hr)
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    gs[hr][a] += __shfl_xor_sync(FULL, gs[hr][a], 1);
                    gs[hr][a] += __shfl_xor_sync(FULL, gs[hr][a], 2);
                }
            if (c == 0) {
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    const int i = i0 + g + 8 * hr;
                    if (i < D) {
                        // n_mid composite: sum_i w_i (n_i + n_i+1) / 2 = sum_i n_i (w_i-1 + w_i) / 2 (w_-1 = w_D-1 = 0)
                        const float wi = i < D - 1 ? __ldg(wts + i) : 0.f;
                        const float coef = 0.5f * ((i > 0 ? __ldg(wts + i - 1) : 0.f) + wi);
                        nacc[0] -= coef * gs[hr][0]; nacc[1] -= coef * gs[hr][1]; nacc[2] -= coef * gs[hr][2];
                        wsum += wi;
                    }
                }
            }
            __syncwarp();                                    // tiles free for the next chunk
        }
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
            nacc[0] += __shfl_xor_sync(FULL, nacc[0], s);
            nacc[1] += __shfl_xor_sync(FULL, nacc[1], s);
            nacc[2] += __shfl_xor_sync(FULL, nacc[2], s);
            wsum += __shfl_xor_sync(FULL, wsum, s);
        }
        if (lane == 0) {
            const float rx = nacc[0] / wsum, ry = nacc[1] / wsum, rz = nacc[2] / wsum;
            const float len = sqrtf(rx * rx + ry * ry + rz * rz) + 1e-7f;
            K.normal[gr * 3 + 0] = rx / len;
            K.normal[gr * 3 + 1] = ry / len;
            K.normal[gr * 3 + 2] = rz / len;
        }
    }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------- ceilings
// Two micro-kernels that isolate the hard per-SM limits of the renderer's formulation on the SAME workload (same rays, same sample
// positions, same tap arithmetic), used by bench.py / DESIGN.md to say how far render_fused_kernel is from what the hardware
// allows for a per-sample gather + MLP -- as opposed to the "every texel read once" HBM figure of the survey's formula:
//   kind 0  gather only : all 16 warps of a CTA run the gather role (ray -> depth -> 12 taps -> 256-bit loads -> weighted sum ->
//           bf16 split -> shared-memory tile).  No MMA, no epilogue.  Ceiling of the tri-plane fetch (L1 wavefronts + L2 misses).
//   kind 1  activations only : 192 MUFU operations per sample (64 x (ex2 + lg2), 32 x (ex2 + rcp)) on register operands with the
//           epilogue's surrounding arithmetic.  Ceiling of the SFU pipe.
namespace {
__global__ void __launch_bounds__(kThreads, 1) gather_floor_kernel(const __grid_constant__ FusedK K, float* __restrict__ sink) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* const sb = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const N3DRender& P = K.p;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int L = 64 / K.gw;                                     // make_fused's lanes per ray
    uint2* const taps = reinterpret_cast<uint2*>(sb + 32768 + warp * kTapBytesPerWarp);
    uint8_t* const f_hi = sb, * const f_lo = sb + 8192;          // one shared tile: the stores are part of the cost, the data is not used
    const int g_begin = (int)((K.total_groups * blockIdx.x) / gridDim.x);
    const int n_groups = (int)((K.total_groups * (blockIdx.x + 1)) / gridDim.x) - g_begin;
    const int passes = P.depth_fine > 0 ? 2 : 1;
    const int T = K.Tc;
    // item = (group, pass, tile, quarter): the same 32-row work unit the gather warps of the renderer process
    const int items = n_groups * passes * T * 4;
    for (int it = warp; it < items; it += kWarps) {
        const int q = it & 3, t = (it >> 2) % T, pass = (it / (4 * T)) % passes, r = it / (4 * T * passes);
        const int row = q * 32 + lane, rs = row / L, j = row & (L - 1);
        const Ray ray = make_ray(K, g_begin + r, rs);
        const int k = t * L + j;
        const bool valid = ray.ok && k < P.depth_coarse;
        // second pass: the fine samples sit near the coarse ones (shifted by half a step) -- same count, same locality
        const float depth = valid ? coarse_depth(K, P.seed + pass, ray.gr, k) + (pass ? 0.5f * K.delta_coarse : 0.f) : 0.f;
        setup_taps(taps, lane, ray.ox + depth * ray.dx, ray.oy + depth * ray.dy, ray.oz + depth * ray.dz, valid, ray.img4, P.PH, P.PW,
                   K.scale);
        __syncwarp();
        gather_rows(P.planes, taps, f_hi, f_lo, q * 32, lane);
        __syncwarp();
    }
    if (sink && threadIdx.x == 0 && blockIdx.x == 0) sink[0] = (float)f_hi[0];
}

__global__ void __launch_bounds__(kThreads, 1) mufu_floor_kernel(long long samples, float* __restrict__ sink) {
    // every thread evaluates whole samples: 64 hidden activations (softplus as in epi1) and 32 colour sigmoids
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nthreads = (long long)gridDim.x * blockDim.x;
    float acc = 0.f;
    for (long long s = tid; s < samples; s += nthreads) {
        float y[32];
#pragma unroll 1
        for (int half = 0; half < 2; ++half) {
#pragma unroll
            for (int c = 0; c < 32; ++c) y[c] = (float)(s & 1023) * 1e-3f + (float)(c + 32 * half) * 0.01f - 0.3f;
            float e[32];
#pragma unroll
            for (int c = 0; c < 32; ++c) e[c] = ex2_approx(fminf(y[c], 126.f));
#pragma unroll
            for (int c = 0; c < 32; ++c) e[c] = lg2_approx(1.f + e[c]);
#pragma unroll
            for (int c = 0; c < 32; ++c) acc += fmaxf(e[c], y[c]);
        }
#pragma unroll
        for (int c = 0; c < 32; ++c) y[c] = (float)(s & 511) * 2e-3f - (float)c * 0.02f;
#pragma unroll
        for (int c = 0; c < 32; ++c) y[c] = ex2_approx(y[c]);
#pragma unroll
        for (int c = 0; c < 32; ++c) y[c] = rcp_approx(1.f + y[c]);
#pragma unroll
        for (int c = 0; c < 32; ++c) acc = fmaf(0.5f, y[c], acc);
    }
    if (sink && acc == 123.456f) sink[0] = acc;
}

// Depth clamp of the composited depth to the depth range (ray_marcher.py:53-54), one range per image: element i belongs to image
// i / per_image and is clamped to its pair of mm [N, 2].  The batch-global clamp is the case of one image.
__global__ void __launch_bounds__(256) depth_clamp_images_kernel(float* __restrict__ depth, int64_t n, int64_t per_image,
                                                                 const float* __restrict__ mm) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t img = i / per_image;
        float d = depth[i];
        if (isnan(d)) d = INFINITY;
        depth[i] = fminf(fmaxf(d, __ldg(mm + 2 * img)), __ldg(mm + 2 * img + 1));
    }
}

constexpr int kMaxD = kMaxT * 64;               // depth samples per pass the fused kernel lays out (3 tiles x 64 lanes per ray)
constexpr int kMaxDFloor = kMaxT * 32;          // the floor micro-kernels know the 16- and 32-lane layouts only

// Images per plane set (N3DRender::views, 0 read as 1): the kernels divide the image index by it.
int plane_views(const N3DRender* p) { return p->views > 1 ? p->views : 1; }

// views >= 0 and N a multiple of it; messages start with `who`.
int check_views(const N3DRender* p, const char* who) {
    N3D_CHECK_ARG(p->views >= 0 && p->N % plane_views(p) == 0, "%s: views = %d must be >= 0 and divide N = %d", who, p->views, p->N);
    return N3D_OK;
}

// Work decomposition of the renderer and of the floor micro-kernels for the workload p; L = lanes per ray (16 up to 48 samples
// per pass, 32 up to 96, else 64).
FusedK make_fused(const N3DRender* p, int& L) {
    const int dmax = p->depth_coarse > p->depth_fine ? p->depth_coarse : p->depth_fine;
    L = dmax <= 48 ? 16 : dmax <= 96 ? 32 : 64;
    FusedK K;
    K.p = *p;
    K.p.views = plane_views(p);
    K.M = p->res * p->res;
    const double span = p->ray_span > 0.0 ? p->ray_span : (double)p->ray_end - (double)p->ray_start;
    K.delta_coarse = (float)(span / (double)(p->depth_coarse - 1));
    K.scale = 2.f / p->box_warp;
    K.Tc = (p->depth_coarse + L - 1) / L;
    K.Tf = (p->depth_fine + L - 1) / L;
    K.gw = 64 / L;                                  // pixel block of a group: 4 x 2, 2 x 2 or 1 x 2
    K.log2gw = L == 16 ? 2 : L == 32 ? 1 : 0;
    const int tiles_x = (p->res + K.gw - 1) / K.gw, tiles_y = (p->res + 1) / 2;
    K.blocks_x = (tiles_x + 3) / 4;
    K.gpi = K.blocks_x * ((tiles_y + 7) / 8) * 32;
    K.total_groups = (long long)p->N * K.gpi;
    return K;
}

// coords != nullptr: arbitrary points [N, Pn, 3].  coords == nullptr: voxel grid of `grid_n`^3 points (image 0), flat indices
// head .. head + Pn - 1, sigma written flipped + trimmed into the [grid_n]^3 output.
int launch_points(const float* planes, int N, int PH, int PW, const float* coords, long long Pn, float box_warp, const float* w0,
                  const float* b0, const float* w1, const float* b1, float* sigma, float* rgb, int grid_n, float cube_length, long long head,
                  int pad, float pad_value, void* stream) {
    PointsK K;
    K.planes = planes; K.N = N; K.PH = PH; K.PW = PW; K.coords = coords; K.Pn = Pn; K.total = (long long)N * Pn;
    K.scale = 2.f / box_warp;
    K.w0 = w0; K.b0 = b0; K.w1 = w1; K.b1 = b1; K.sigma = sigma; K.rgb = rgb;
    K.grid_n = grid_n; K.pad = pad; K.pad_value = pad_value; K.head = head;
    K.voxel_size = 0.f; K.org0 = K.org1 = K.org2 = 0.f;
    if (!coords) {       // create_samples: voxel_origin = [0,0,0] - cube_length / 2 (float64), voxel_size = cube_length / (N - 1); both enter
                         // the float32 tensor expression as scalars, i.e. rounded to float32
        K.voxel_size = (float)((double)cube_length / (double)(grid_n - 1));
        K.org0 = K.org1 = K.org2 = (float)(0.0 - (double)cube_length / 2.0);
    }
    const int smem = kSmemBytes + 1024;
    if (int rc = n3d_smem_optin(rgb ? (const void*)points_fused_kernel<true> : (const void*)points_fused_kernel<false>, smem, "n3d_sample_points"))
        return rc;
    const N3DDeviceState* D = n3d_device_state();
    if (!D) return N3D_ERR_CUDA;
    const long long tiles = (K.total + 127) / 128;
    const int grid = (int)(tiles < D->num_sms ? tiles : D->num_sms);
    if (rgb) points_fused_kernel<true><<<grid, kThreads, smem, (cudaStream_t)stream>>>(K);
    else points_fused_kernel<false><<<grid, kThreads, smem, (cudaStream_t)stream>>>(K);
    N3D_CHECK_LAUNCH("n3d_sample_points");
    return N3D_OK;
}
}  // namespace

namespace {
// Argument checks of n3d_render_rays / n3d_render_rays_normals (messages start with `who`).
int check_render(const N3DRender* p, const char* who) {
    N3D_CHECK_ARG(p && p->planes && p->cam2world && p->intrinsics && p->w0 && p->b0 && p->w1 && p->b1 && p->rgb && p->depth && p->wsum,
                  "%s: null pointer", who);
    N3D_CHECK_ARG(((uintptr_t)p->planes & 31) == 0, "%s: planes must be 32-byte aligned", who);      // 256-bit texel loads
    if (p->depth_coarse > kMaxD || p->depth_fine > kMaxD) {
        n3d_set_error("%s: depth resolutions (%d, %d) above %d samples per pass are not supported", who, p->depth_coarse, p->depth_fine, kMaxD);
        return N3D_ERR_UNSUPPORTED;
    }
    N3D_CHECK_ARG(p->depth_coarse >= 4 && p->depth_fine >= 0, "%s: depth resolutions (%d, %d): need coarse >= 4, fine >= 0", who,
                  p->depth_coarse, p->depth_fine);
    if (int rc = check_views(p, who)) return rc;
    N3D_CHECK_ARG(p->depth_range_per_image == 0 || p->depth_range_per_image == 1, "%s: depth_range_per_image = %d must be 0 or 1", who,
                  p->depth_range_per_image);
    N3D_CHECK_ARG(!p->depth_range_per_image || p->depth_minmax, "%s: depth_range_per_image = 1 needs depth_minmax [N, 2]", who);
    N3D_CHECK_ARG((long long)(p->N / plane_views(p)) * 3 * p->PH * p->PW * 128 < (1ll << 32), "%s: plane tensor too large for 32-bit texel offsets",
                  who);
    N3D_CHECK_ARG(p->res >= 1 && p->N >= 1 && p->ray_start > 0.f && p->ray_end > p->ray_start && p->box_warp > 0.f, "%s: bad ray setup", who);
    return N3D_OK;
}

// render_fused_kernel<L, kExport> on the checked workload p; kExport writes the per-ray samples to `samples`.
template <bool kExport>
int launch_render(const N3DRender* p, float* samples, const char* who, void* stream) {
    int L;
    FusedK K = make_fused(p, L);
    K.samples = samples;
    const int smem = kSmemBytes + 1024;
    const void* const fn = L == 16 ? (const void*)render_fused_kernel<16, kExport>
                         : L == 32 ? (const void*)render_fused_kernel<32, kExport> : (const void*)render_fused_kernel<64, kExport>;
    if (int rc = n3d_smem_optin(fn, smem, who)) return rc;
    const N3DDeviceState* D = n3d_device_state();
    if (!D) return N3D_ERR_CUDA;
    const int grid = (int)(K.total_groups < D->num_sms ? K.total_groups : D->num_sms);
    if (L == 16) render_fused_kernel<16, kExport><<<grid, kThreads, smem, (cudaStream_t)stream>>>(K);
    else if (L == 32) render_fused_kernel<32, kExport><<<grid, kThreads, smem, (cudaStream_t)stream>>>(K);
    else render_fused_kernel<64, kExport><<<grid, kThreads, smem, (cudaStream_t)stream>>>(K);
    N3D_CHECK_LAUNCH(who);
    return N3D_OK;
}
}  // namespace

extern "C" int n3d_render_rays(const N3DRender* p, void* stream) {
    if (int rc = check_render(p, "n3d_render_rays")) return rc;
    return launch_render<false>(p, nullptr, "n3d_render_rays", stream);
}

namespace {
// normals_fused_kernel over the samples render_fused_kernel<L, true> left in `workspace`.
int launch_normals(const N3DRender* p, const float* workspace, float* normal, const char* who, void* stream) {
    NormalsK K;
    K.p = *p;
    K.p.views = plane_views(p);
    K.D = p->depth_fine > 0 ? p->depth_coarse + p->depth_fine : p->depth_coarse;
    K.scale = 2.f / p->box_warp;
    K.rays = (long long)p->N * p->res * p->res;
    K.samples = workspace;
    K.normal = normal;
    if (int rc = n3d_smem_optin((const void*)normals_fused_kernel, kNSmemBytes, who)) return rc;
    const N3DDeviceState* D = n3d_device_state();
    if (!D) return N3D_ERR_CUDA;
    const long long blocks = (K.rays + kNWarps - 1) / kNWarps;
    const int grid = (int)(blocks < 2ll * D->num_sms ? blocks : 2ll * D->num_sms);
    normals_fused_kernel<<<grid, kNThreads, kNSmemBytes, (cudaStream_t)stream>>>(K);
    N3D_CHECK_LAUNCH(who);
    return N3D_OK;
}
}  // namespace

extern "C" int n3d_render_rays_normals(const N3DRender* p, float* normal, float* workspace, void* stream) {
    const char* who = "n3d_render_rays_normals";
    if (int rc = check_render(p, who)) return rc;
    N3D_CHECK_ARG(normal && workspace, "%s: null pointer", who);
    if (int rc = launch_render<true>(p, workspace, who, stream)) return rc;
    return launch_normals(p, workspace, normal, who, stream);
}

extern "C" int n3d_render_normals_pass(const N3DRender* p, const float* workspace, float* normal, void* stream) {
    const char* who = "n3d_render_normals_pass";
    if (int rc = check_render(p, who)) return rc;
    N3D_CHECK_ARG(normal && workspace, "%s: bad args", who);
    return launch_normals(p, workspace, normal, who, stream);
}

extern "C" int n3d_render_floor(const N3DRender* p, int kind, float* sink, void* stream) {
    N3D_CHECK_ARG(p && p->planes && p->cam2world && p->intrinsics && (kind == 0 || kind == 1), "n3d_render_floor: bad args");
    N3D_CHECK_ARG(p->depth_coarse >= 4 && p->depth_coarse <= kMaxDFloor && p->depth_fine >= 0 && p->depth_fine <= kMaxDFloor,
                  "n3d_render_floor: depth resolutions");
    if (int rc = check_views(p, "n3d_render_floor")) return rc;
    int L;
    const FusedK K = make_fused(p, L);
    const N3DDeviceState* D = n3d_device_state();
    if (!D) return N3D_ERR_CUDA;
    if (kind == 0) {
        const int smem = 32768 + kWarps * kTapBytesPerWarp + 1024;
        if (int rc = n3d_smem_optin((const void*)gather_floor_kernel, smem, "n3d_render_floor")) return rc;
        gather_floor_kernel<<<(int)(K.total_groups < D->num_sms ? K.total_groups : D->num_sms), kThreads, smem, (cudaStream_t)stream>>>(K, sink);
    } else {
        const long long samples = (long long)p->N * K.M * (p->depth_coarse + p->depth_fine);
        mufu_floor_kernel<<<D->num_sms, kThreads, 0, (cudaStream_t)stream>>>(samples, sink);
    }
    N3D_CHECK_LAUNCH("n3d_render_floor");
    return N3D_OK;
}

extern "C" int n3d_depth_clamp(float* depth, int64_t n, const float* depth_minmax, void* stream) {
    N3D_CHECK_ARG(depth && depth_minmax && n >= 0, "n3d_depth_clamp: bad args");
    if (n == 0) return N3D_OK;
    depth_clamp_images_kernel<<<n3d_grid(n, 256), 256, 0, (cudaStream_t)stream>>>(depth, n, n, depth_minmax);
    N3D_CHECK_LAUNCH("n3d_depth_clamp");
    return N3D_OK;
}

extern "C" int n3d_depth_clamp_images(float* depth, int N, int64_t per_image, const float* depth_minmax, void* stream) {
    N3D_CHECK_ARG(depth && depth_minmax && N >= 0 && per_image >= 0, "n3d_depth_clamp_images: bad args (N = %d, per_image = %lld)", N,
                  (long long)per_image);
    const int64_t n = (int64_t)N * per_image;
    if (n == 0) return N3D_OK;
    depth_clamp_images_kernel<<<n3d_grid(n, 256), 256, 0, (cudaStream_t)stream>>>(depth, n, per_image, depth_minmax);
    N3D_CHECK_LAUNCH("n3d_depth_clamp_images");
    return N3D_OK;
}

extern "C" int n3d_sample_points(const float* planes, int N, int PH, int PW, const float* coords, int64_t P, float box_warp,
                                 const float* w0, const float* b0, const float* w1, const float* b1, float* sigma, float* rgb,
                                 void* stream) {
    N3D_CHECK_ARG(planes && coords && w0 && b0 && w1 && b1 && sigma && N >= 1 && P >= 1 && box_warp > 0.f, "n3d_sample_points: bad args");
    N3D_CHECK_ARG((long long)N * 3 * PH * PW * 128 < (1ll << 32), "n3d_sample_points: plane tensor too large for 32-bit texel offsets");
    N3D_CHECK_ARG(((uintptr_t)planes & 31) == 0, "n3d_sample_points: planes must be 32-byte aligned");       // 256-bit texel loads
    N3D_CHECK_ARG(((uintptr_t)rgb & 7) == 0, "n3d_sample_points: rgb must be 8-byte aligned");              // float2 stores
    return launch_points(planes, N, PH, PW, coords, P, box_warp, w0, b0, w1, b1, sigma, rgb, 0, 0.f, 0, 0, 0.f, stream);
}

extern "C" int n3d_sample_grid(const float* planes, int PH, int PW, int grid_n, float cube_length, float box_warp, int64_t head, int64_t count,
                               int pad, float pad_value, const float* w0, const float* b0, const float* w1, const float* b1, float* sigma_grid,
                               void* stream) {
    N3D_CHECK_ARG(planes && w0 && b0 && w1 && b1 && sigma_grid && grid_n >= 2 && cube_length > 0.f && box_warp > 0.f, "n3d_sample_grid: bad args");
    N3D_CHECK_ARG(head >= 0 && count >= 1 && head + count <= (int64_t)grid_n * grid_n * grid_n, "n3d_sample_grid: index range outside the grid");
    N3D_CHECK_ARG(pad >= 0 && 2 * pad <= grid_n, "n3d_sample_grid: bad trim width");
    N3D_CHECK_ARG((long long)3 * PH * PW * 128 < (1ll << 32), "n3d_sample_grid: plane tensor too large for 32-bit texel offsets");
    N3D_CHECK_ARG(((uintptr_t)planes & 31) == 0, "n3d_sample_grid: planes must be 32-byte aligned");         // 256-bit texel loads
    return launch_points(planes, 1, PH, PW, nullptr, count, box_warp, w0, b0, w1, b1, sigma_grid, nullptr, grid_n, cube_length, head, pad,
                         pad_value, stream);
}
