// Implicit-GEMM convolution on Hopper warpgroup tensor cores (wgmma, sm_90a) -- the dense contraction of every conv layer of the
// generator (modulated 3x3 / 1x1, transposed-conv parity classes, stride-2 convs, ToRGB).
//
//   M = 128 output pixels per tile (TN x TH x TW patch), N = block_n output channels, K = taps x Cin.
//   A (activations, NHWC bf16, split hi/lo) is fetched per (tap, 64- or 32-channel chunk) as one 4-D TMA box whose
//   coordinates are shifted by the tap offset; out-of-range rows/columns are zero-filled by TMA, which *is* the
//   convolution padding.  B (weights [T, Cout, Cin] bf16 hi/lo) is a 3-D TMA box.  Both land in shared memory in the
//   K-major SWIZZLE_128B / SWIZZLE_64B layout that wgmma consumes directly.
//   Precision: fp32 = hi + lo with bf16 hi, lo; acc += Ahi*Bhi + Ahi*Blo + Alo*Bhi (3 MMAs, fp32 accumulate in registers)
//   reproduces an fp32 convolution to ~2^-16 relative -- inside the 1e-3 end-to-end budget where single-pass
//   bf16/fp16/tf32 is not (SURVEY.md section 7 "Precision vs tensor cores").
//   Warp roles (384 threads, persistent over work items): warps 0-7 = two ping-pong consumer warpgroups; the CTA's work items
//   alternate between them, and each owns all 128 rows of its tiles: wgmma into a register accumulator (two m64 halves), then the
//   fused epilogue (demod/noise/bias/lrelu/clamp -> next layer's modulation -> bf16 split / fp32 stores) through a small
//   shared-memory transpose (thread = tile row, one 64-row half at a time), overlapping the other warpgroup's MMAs; raw fp32 output
//   (mode 1) leaves through TMA stores instead (store_raw_tma).  Warpgroup 2 = TMA
//   producer (one lane), which keeps filling the stage ring during the epilogue.  setmaxnreg lowers the producer to 24 registers
//   and raises the consumers to 240 (2 x 128 x 240 + 128 x 24 = 384 x 168): ptxas allocates each role's code to its own budget (the launch figure it reports is 168).
//   Launches with wide tiles run as 2-CTA clusters: the two CTAs take neighbouring M tiles of the same n-tile and K steps, and
//   each loads half of the shared weight tile, multicast into both (decode_tile, the producer, release_stage, launch_conv).
//   fp16 instances (template F16, N3DConvGemm::f16): fp16 operands, one wgmma...f32.f16.f16 per k16 step, a stage of one A and one
//   B tile (so the same ring holds twice the K steps), and fp16 single outputs in place of the split pairs.  They serve the opt-in
//   fp16 super-resolution head; the bf16 instances and their launch rule do not depend on them.
#include <cstring>
#include "common.cuh"
#include <cuda.h>
#include "tc_ptx.cuh"

namespace {
using namespace n3d_tc;

constexpr int kBlockM = 128;
// K per pipeline stage (block_k, a template parameter): 64 bf16 (128-byte rows, SWIZZLE_128B) or 32 bf16 (64-byte rows,
// SWIZZLE_64B).  32 is used for Cin % 64 == 32 (the 32-channel feature images: no TMA box hangs over the channel extent) and
// wherever 64-channel stages would leave fewer than kMinStages in the ring (block_n 96 and 128).
constexpr int kConsumerThreads = 256;         // two ping-pong warpgroups of 128 tile rows each
constexpr int kThreads = kConsumerThreads + 128;   // + the producer warpgroup (one TMA lane)
constexpr int kMaxBlockN = 128;
constexpr int kMinStages = 4;
constexpr int kMaxStages = 8;
constexpr int kMinTiles = 64;                 // see the block_n choice in launch_conv
constexpr int kMinTilesSplit = 128;           // same for split-K launches
constexpr int kStageArrays = 8;               // dcoef | bias | style0 | style1 | up to 4 modulated ToRGB weight rows
constexpr int kXStride = 36;                  // floats per row of the accumulator transpose buffer (32 columns + pad)
constexpr int kStoreBoxBytes = 64 * 32 * 4;   // one TMA store box of the raw fp32 output: 64 tile rows x 32 channels
// Per-warpgroup epilogue area (1024-byte aligned), used one of two ways:
//   per-thread stores: staged vectors | accumulator transpose [64][kXStride] | ToRGB partial sums [64][4]
//   TMA stores of the raw output (KParams::tma_store): two store boxes, one being filled while the other is read by the TMA
constexpr int kThreadEpiBytes = kStageArrays * kMaxBlockN * 4 + 64 * kXStride * 4 + 64 * 4 * 4;
constexpr int kEpiBytes = kThreadEpiBytes > 2 * kStoreBoxBytes ? kThreadEpiBytes : 2 * kStoreBoxBytes;
static_assert(kEpiBytes % 1024 == 0, "the store boxes of both warpgroups are SWIZZLE_128B atoms");
// shared memory left for the stage ring: opt-in maximum - both epilogue areas - barriers - 1024-byte alignment slack
constexpr int kRingBytes = 227 * 1024 - 2 * kEpiBytes - 1024 - 256;
constexpr int kMaxSubs = 9;                   // a stride-2 transposed conv: 4 parity-class interiors + 5 edge strips / corner
constexpr int kMaxBoxes = 4;                  // distinct A box shapes (tile geometries) of one launch

struct KParams {
    CUtensorMap tmA[kMaxBoxes][2];   // A (hi, lo) per tile geometry: box (block_k, TW, TH, TN) of the sub-problems using it
    CUtensorMap tmB_hi, tmB_lo;
    int N, Cout;
    int tiles_n;
    // sub-problems sharing operands and epilogue (the output-parity classes of a stride-2 transposed conv and their edges), each
    // with its own tile geometry (TW*TH*TN == 128, all powers of two) over the M-space rectangle [y0, y_end) x [x0, x_end)
    int nsub, nint, groups, nbox;    // the first nint sub-problems are interleaved (see decode_tile), groups: see unit_item
    struct Sub { int tap_begin, ntaps, TW, TH, TN, box, tiles_x, tiles_y, tiles_m, y0, x0, y_end, x_end, oy_off, ox_off, tile_end; } sub[kMaxSubs];
    int cluster, b_rows;             // CTAs per cluster (1 or 2): a pair shares the weight tile, each loads b_rows = block_n / cluster of its rows
    int splits; long long split_stride;   // split-K: work item = (tile, K slice); slice s writes its raw partial sums to out_f32 + s * split_stride
    int block_n, stages, stage_bytes, b_bytes, a_bytes;
    int item_tiles;                  // n-tiles per work item: tiles_n for the fused ToRGB (all channels of a pixel), else 1
    int total_items;                 // sub[nsub - 1].tile_end * splits / item_tiles (a kernel parameter: the producer has no register for it)
    int cin_chunks, nprod, a_img_stride;
    N3DConvTap taps[9];
    int mode;
    const float* dcoef; const float* bias; const float* noise; int64_t noise_nstride;
    float gain, slope, clamp;
    N3DSplitOut out[2];
    float* out_f32; int f32_cstride, f32_coff, f32_nchw, f32_accumulate;
    N3DFusedRgb rgb;                 // optional fused ToRGB (<= 4 image channels), see include/next3d_b200.h
    int oy_mul, ox_mul, OH, OW;
    int* err_flag;
    // raw fp32 output of each sub-problem (tma_store): dims (Cout, x, y, N, K slice) in the sub-problem's M-space coordinates,
    // clipped where the per-thread stores test `valid`; box (min(32, block_n), TW, the 64-row half of TH x TN, 1)
    // (last: placed before the scalar fields, it cost the 128-wide instances spills)
    CUtensorMap tmC[kMaxSubs];
    int tma_store;
};
static_assert(sizeof(KParams) <= 4096, "KParams is passed as a kernel parameter");

// mode-0 launches always have a single sub-problem
__device__ __forceinline__ int staged_rgb_channels(const KParams& P) { return (P.rgb.out && P.sub[0].TN == 1 && P.mode == 0 && P.item_tiles == P.tiles_n) ? P.rgb.channels : 0; }

struct TileInfo { int sub, tn, x0, y0, n0, split; bool pad; };
// Tiles are numbered sub-problem-major, n-tile minor, except that the first nint sub-problems (the four parity classes of a
// transposed conv over the same input rectangle, one tile geometry) are interleaved class-minor: the classes of one M tile and
// n-tile are consecutive tiles.  They share one tile_end, so the search below steps over all of them at once.
// In a 2-CTA cluster a tile number stands for a pair of M tiles: CTA rank r takes M tile 2m + r with the same sub-problem,
// n-tile and K slice, so both CTAs run the same K-step sequence on the same weight tiles.  A sub-problem with an odd number of
// M tiles ends in a pad tile: it repeats its partner's A tile (so that both CTAs still load and consume the same stages) and
// its epilogue writes nothing.
__device__ __forceinline__ TileInfo decode_tile(const KParams& P, int tile) {
    const int split = tile % P.splits;                         // K slices of one tile are neighbouring work items (run concurrently)
    tile /= P.splits;
    int sidx = 0, begin = 0;
    while (sidx + 1 < P.nsub && tile >= P.sub[sidx].tile_end) { begin = P.sub[sidx].tile_end; ++sidx; }
    int local = tile - begin;
    if (sidx < P.nint) { sidx = local % P.nint; local /= P.nint; }
    const KParams::Sub& S = P.sub[sidx];
    TileInfo t;
    t.sub = sidx;
    t.tn = local % P.tiles_n;
    int tm = local / P.tiles_n;
    t.pad = false;
    if (P.cluster > 1) {
        tm = tm * P.cluster + (int)cluster_ctarank();
        t.pad = tm >= S.tiles_m;
        if (t.pad) tm -= 1;
    }
    t.x0 = S.x0 + (tm % S.tiles_x) * S.TW;
    t.y0 = S.y0 + ((tm / S.tiles_x) % S.tiles_y) * S.TH;
    t.n0 = (tm / (S.tiles_x * S.tiles_y)) * S.TN;
    t.split = split;
    return t;
}

// Work distribution: clusters take units round-robin (unit c, then + the number of clusters, ...; a launch without clusters has
// one per CTA), and both CTAs of a cluster take the same units.  The first P.groups units are P.nint consecutive items each (the
// parity classes of one M tile and n-tile: they read the same input rows, so all but the first read them from L2, and every such
// unit costs the same); every later unit is one item.  With P.groups == 0 and no clusters a CTA's items are
// blockIdx.x + k * gridDim.x.
__device__ __forceinline__ int unit_item(const KParams& P, int unit) { return unit < P.groups ? unit * P.nint : unit + P.groups * (P.nint - 1); }
__device__ __forceinline__ int next_item(const KParams& P, int item) {      // this CTA's work item after `item`
    const int grouped = P.groups * P.nint;
    if (item < grouped && (item + 1) % P.nint != 0) return item + 1;
    return unit_item(P, (item < grouped ? item / P.nint : item - grouped + P.groups) + num_clusters_x());
}

// A consumer warp releases a stage: it arrives on the stage's empty barrier in every CTA of the cluster, since the producer of
// each CTA multicasts its half of the weight tile into both.
__device__ __forceinline__ void release_stage(const KParams& P, uint32_t empty_bar) {
    if (P.cluster == 1) mbar_arrive(empty_bar);
    else { mbar_arrive_cluster(empty_bar, 0); mbar_arrive_cluster(empty_bar, 1); }
}

// K-step range [kb, ke) of a work item: all taps x channel chunks, or the item's slice of them under split-K.
__device__ __forceinline__ void k_range(const KParams& P, const TileInfo& t, int& kb, int& ke) {
    const int nsteps = P.sub[t.sub].ntaps * P.cin_chunks, per = (nsteps + P.splits - 1) / P.splits;
    kb = t.split * per;
    ke = min(nsteps, kb + per);
}

// Main loop of one tile: one stage = one (tap, channel chunk); a stage is released once its wgmmas retired (wait_group 1 after
// the next stage's wgmmas are issued, so that the tensor cores always have one group queued).  Each of the warpgroup's 4 warps
// arrives on the stage's empty barrier (of both CTAs in a cluster).
template <int BN, int BK, int NPROD, bool F16>
__device__ __forceinline__ void tile_mainloop(const KParams& P, float (&acc0)[BN / 2], float (&acc1)[BN / 2], int ksteps, uint32_t smem_base,
                                              uint32_t bar_base, int lane, int& s, uint32_t& ph) {
    const uint32_t a_bytes = (uint32_t)P.a_bytes, b_bytes = (uint32_t)P.b_bytes, stage_bytes = (uint32_t)P.stage_bytes;
    const uint32_t empty_base = bar_base + 8u * (uint32_t)P.stages;
    const uint32_t b_off = F16 ? a_bytes : 2u * a_bytes;               // stage: A hi [| A lo] | B hi [| B lo]
    uint32_t sa = smem_base + (uint32_t)s * stage_bytes;
    mbar_wait(bar_base + 8u * (uint32_t)s, ph, P.err_flag, 3);           // first stage (ksteps >= 1): overwrite the accumulator
    stage_mma<BN, BK, NPROD, true, F16>(acc0, acc1, sa, sa + a_bytes, sa + b_off, sa + b_off + b_bytes);
    int prev_s = s;
    if (++s == P.stages) { s = 0; ph ^= 1u; }
    for (int ks = 1; ks < ksteps; ++ks) {
        sa = smem_base + (uint32_t)s * stage_bytes;
        mbar_wait(bar_base + 8u * (uint32_t)s, ph, P.err_flag, 3);
        stage_mma<BN, BK, NPROD, false, F16>(acc0, acc1, sa, sa + a_bytes, sa + b_off, sa + b_off + b_bytes);
        wgmma_wait<1>();
        __syncwarp();
        if (lane == 0) release_stage(P, empty_base + 8u * (uint32_t)prev_s);
        prev_s = s;
        if (++s == P.stages) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) release_stage(P, empty_base + 8u * (uint32_t)prev_s);
}

// Raw fp32 epilogue (KParams::tma_store): 64-row half h of a tile, min(32, BN) channels at a time, goes from the accumulator
// fragments into one of the warpgroup's two store boxes (the layout of the tensor map's box, swizzled like it so that the
// fragment writes do not conflict) and out with one TMA store, which the leader thread issues and commits.  Before the barrier
// that releases a box to the TMA, the leader waits until the previous box has been read, so the other box may be refilled
// right after the barrier while this one is read; the global writes stay in flight.  Clipping by the tensor map does what
// `valid` does in the per-thread stores; pad tiles store nothing.
template <int BN>
__device__ __forceinline__ void store_raw_tma(const KParams& P, const float (&acc)[BN / 2], const TileInfo& ti, int h,
                                              bool leader, int bar_id, uint32_t boxes) {
    constexpr int BC = BN < 32 ? BN : 32;                  // channels per box
    constexpr uint32_t kRow = BC * 4;                      // bytes per box row: 128 (SWIZZLE_128B) or 64 (SWIZZLE_64B)
    // Fragment element i of this thread: row r = r0 + 8 * ((i >> 1) & 1), 16-byte chunk 2 * ((i >> 2) & 3) + (lane & 3) / 2 of the
    // box row, 8 bytes in.  The TMA swizzle of a 1024-byte aligned box XORs the chunk index with row address bits 7.. (the same for
    // r0 and r0 + 8), so the byte offset is sw ^ (((i >> 2) & 3) << 5), plus 8 rows for the second row.
    // (the thread's position is read here, not passed in: with values derived from it outside the item loop the 128-wide
    // instances spill)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t r0 = 16 * (warp & 3) + (lane >> 2);
    const uint32_t sw = r0 * kRow + ((((uint32_t)(lane & 3) >> 1) ^ ((r0 * kRow >> 7) & (kRow / 16 - 1))) << 4) + (lane & 1) * 8;
#pragma unroll
    for (int cc = 0; cc < BN / BC; ++cc) {
        // a tile fills an even number of boxes, so the two alternate across tiles as well
        const uint32_t box = boxes + (uint32_t)((h * (BN / BC) + cc) & 1) * (uint32_t)kStoreBoxBytes;
#pragma unroll
        for (int e = 0; e < BC / 2; e += 2) {
            const int i = cc * (BC / 2) + e;
            const uint32_t off = (sw ^ (uint32_t)(((i >> 2) & 3) << 5)) + (uint32_t)((i >> 1) & 1) * 8u * kRow;
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(box + off), "f"(acc[i]), "f"(acc[i + 1]) : "memory");
        }
        fence_proxy_async_smem();
        if (leader) bulk_wait_read_all();
        asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
        if (leader) {
            if (!ti.pad) {
                // the half is the second half of the tile's images, or of its rows when it has one image (TH >= 8 then)
                const KParams::Sub& S = P.sub[ti.sub];
                const int y = ti.y0 + (S.TN > 1 ? 0 : h * (S.TH / 2)), n = ti.n0 + (S.TN > 1 ? h * (S.TN / 2) : 0);
                tma_store_5d(&P.tmC[ti.sub], box, ti.tn * P.block_n + cc * BC, ti.x0, y, n, ti.split);
            }
            bulk_commit_group();
        }
    }
}

// ---------------------------------------------------------------------------------------------- the kernel
// Body of conv_gemm_kernel (bf16 operands) and conv_gemm_f16_kernel (F16: fp16 operands and outputs).
template <int BN, int BK, bool F16>
__device__ __forceinline__ void conv_gemm_body(const KParams& P) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // dynamic smem base is only guaranteed 16-B aligned: round up to 1024 (SWIZZLE_128B atoms)
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    // the stage ring (whole KiB per stage), the two warpgroups' epilogue areas, then the barriers full[stages], empty[stages]
    const uint32_t epi_base = smem_base + (uint32_t)P.stages * (uint32_t)P.stage_bytes;
    const uint32_t bar_base = epi_base + 2u * (uint32_t)kEpiBytes;
    auto full_bar = [&](int s) { return bar_base + 8u * (uint32_t)s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (uint32_t)(P.stages + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == kConsumerThreads / 32 && lane == 0) {
        tma_prefetch_desc(&P.tmB_hi);
        if (P.nprod == 3) tma_prefetch_desc(&P.tmB_lo);
        for (int b = 0; b < P.nbox; ++b) {
            tma_prefetch_desc(&P.tmA[b][0]);
            if (P.nprod == 3) tma_prefetch_desc(&P.tmA[b][1]);
        }
        // one stage feeds one warpgroup in each CTA of the cluster, and all of them must be done before either producer refills it
        for (int s = 0; s < P.stages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 4 * P.cluster); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // the partner's first multicast and remote arrivals need this CTA's barriers initialised
    if (P.cluster > 1) cluster_sync();
    else __syncthreads();

    // work item = item_tiles consecutive tiles (n-tile minor: all n-tiles of one M tile for the fused ToRGB), one CTA each
    const int total_items = P.total_items;

    if (warp >= kConsumerThreads / 32) {
        // ===================================================== TMA producer
        asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
        if (warp == kConsumerThreads / 32 && lane == 0) {
            int s = 0; uint32_t ph = 0;
            // the full barrier counts the whole stage: this CTA's A tile and both halves of the B tile (one multicast by each CTA)
            const uint32_t tx_bytes = (uint32_t)(P.nprod == 3 ? 2 : 1) * (uint32_t)(P.a_bytes + P.b_bytes);
            for (int item = unit_item(P, cluster_idx_x()); item < total_items; item = next_item(P, item))
            for (int tile = item * P.item_tiles; tile < (item + 1) * P.item_tiles; ++tile) {
                const TileInfo ti = decode_tile(P, tile);
                const int tn = ti.tn, x0 = ti.x0, y0 = ti.y0, n0 = ti.n0;
                const int tap_begin = P.sub[ti.sub].tap_begin;
                const CUtensorMap* const tmA = P.tmA[P.sub[ti.sub].box];
                int kb, ke;
                k_range(P, ti, kb, ke);
                for (int idx = kb; idx < ke; ++idx) {
                    const int t = idx / P.cin_chunks, kc = idx - t * P.cin_chunks;
                    const N3DConvTap tap = P.taps[tap_begin + t];
                    mbar_wait(empty_bar(s), ph ^ 1u, P.err_flag, 1);
                    const uint32_t sa = smem_base + (uint32_t)s * (uint32_t)P.stage_bytes;
                    const uint32_t fb = full_bar(s);
                    mbar_expect_tx(fb, tx_bytes);
                    const int img = n0 + (int)tap.img_off * P.a_img_stride;
                    tma_load_4d(sa, &tmA[0], fb, kc * BK, x0 + tap.dx, y0 + tap.dy, img);
                    if (P.nprod == 3) tma_load_4d(sa + P.a_bytes, &tmA[1], fb, kc * BK, x0 + tap.dx, y0 + tap.dy, img);
                    // B: rows [r * b_rows, (r + 1) * b_rows) of the n-tile (all of them without a cluster, r = 0), multicast to the
                    // same offset in both CTAs of a cluster.  The rank is read here, not kept: the producer's 24 registers hold no
                    // further live value without spilling.
                    const int r = (int)cluster_ctarank();
                    const uint32_t sb = sa + (F16 ? 1 : 2) * P.a_bytes + (uint32_t)(r * P.b_rows * BK * 2);
                    const int brow = tn * P.block_n + r * P.b_rows;
                    if (P.cluster == 1) {
                        tma_load_3d(sb, &P.tmB_hi, fb, kc * BK, brow, tap.wtap);
                        if (P.nprod == 3) tma_load_3d(sb + P.b_bytes, &P.tmB_lo, fb, kc * BK, brow, tap.wtap);
                    } else {
                        tma_load_3d_multicast(sb, &P.tmB_hi, fb, kc * BK, brow, tap.wtap, 0x3);
                        if (P.nprod == 3) tma_load_3d_multicast(sb + P.b_bytes, &P.tmB_lo, fb, kc * BK, brow, tap.wtap, 0x3);
                    }
                    if (++s == P.stages) { s = 0; ph ^= 1u; }
                }
            }
        }
    } else {
        // ===================================================== consumers: ping-pong, warpgroup g = work items 2i + g of this CTA
        asm volatile("setmaxnreg.inc.sync.aligned.u32 240;");
        const int g = warp >> 2;
        const int gtid = threadIdx.x & 127;                    // thread index inside the warpgroup
        const int xrow = gtid & 63, half = gtid >> 6;          // epilogue: tile row 64h + xrow, columns 16 * half of each 32-column chunk
        uint8_t* const epi = smem_raw + (epi_base - smem_u32(smem_raw)) + (uint32_t)g * (uint32_t)kEpiBytes;
        float* const stg = reinterpret_cast<float*>(epi);                                   // [kStageArrays][kMaxBlockN]
        float* const xbuf = stg + kStageArrays * kMaxBlockN;                                // [64][kXStride]
        float* const rbuf = xbuf + 64 * kXStride;                                           // [64][4]
        const int nrgb = staged_rgb_channels(P);
        const bool staged = (P.sub[0].TN == 1) && (P.mode == 0);
        int s = 0; uint32_t ph = 0;
        // fused ToRGB: the partial sums of a pixel run over all n-tiles of its work item, in column order
        float raccs[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
        // The producer fills the ring in the CTA's item order; the items alternate between the warpgroups, so one warpgroup's
        // epilogue runs while the other's MMAs run.  A warpgroup steps its ring position past the other one's K steps.
        auto skip_item = [&](int item) {
            for (int tile = item * P.item_tiles; tile < (item + 1) * P.item_tiles; ++tile) {
                int kb, ke;
                k_range(P, decode_tile(P, tile), kb, ke);
                const int pos = s + (ke - kb);
                ph ^= (uint32_t)((pos / P.stages) & 1);
                s = pos % P.stages;
            }
        };
        // Order barrier (named barriers 3 + g): a warpgroup starts an item's main loop only after the other warpgroup has issued
        // the main loop of the item before it.  Every stage of that item has then been waited on, so the first stage this warpgroup
        // waits for is at most one phase ahead of its full barrier (a parity wait cannot tell phases two apart).
        const int first_item = unit_item(P, cluster_idx_x());
        int item = first_item;
        if (g == 1) {
            if (item < total_items) skip_item(item);
            item = next_item(P, item);
        }
        for (; item < total_items; item = next_item(P, item)) {
        const int other_item = next_item(P, item);             // the other warpgroup's next item
        if (item != first_item) asm volatile("bar.sync %0, 256;" ::"r"(3 + g) : "memory");
        for (int tile = item * P.item_tiles; tile < (item + 1) * P.item_tiles; ++tile) {
            const TileInfo ti = decode_tile(P, tile);
            const int tn = ti.tn, n0 = ti.n0;
            if (staged) {
                // the warpgroup is done with the previous tile's vectors before they are overwritten
                asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
                for (int i = gtid; i < 4 * P.block_n; i += 128) {
                    const int arr = i / P.block_n, c = i - arr * P.block_n, co = tn * P.block_n + c;
                    float val = arr == 1 ? 0.f : 1.f;
                    if (co < P.Cout && n0 < P.N) {
                        const float* src = arr == 0 ? P.dcoef : arr == 1 ? P.bias : (arr == 2 ? P.out[0].style : P.out[1].style);
                        if (src) val = __ldg(src + (arr == 1 ? (int64_t)co : (int64_t)n0 * P.Cout + co));
                    }
                    stg[arr * kMaxBlockN + c] = val;
                }
                for (int i = gtid; i < nrgb * P.block_n; i += 128) {          // fused ToRGB: W_rgb[c, co] * style_rgb[n, co]
                    const int c = i / P.block_n, cl = i - c * P.block_n, co = tn * P.block_n + cl;
                    float val = 0.f;
                    if (co < P.Cout && n0 < P.N) val = __ldg(P.rgb.weight + (int64_t)c * P.Cout + co) * __ldg(P.rgb.style + (int64_t)n0 * P.Cout + co);
                    stg[(4 + c) * kMaxBlockN + cl] = val;
                }
                asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
            }

            // ---- main loop (nprod and the accumulator overwrite of the first stage are fixed outside the instruction stream)
            int kb, ke;
            k_range(P, ti, kb, ke);
            float accs[2][BN / 2];                                 // rows 0-63 | 64-127; the first stage overwrites them
            if (F16) tile_mainloop<BN, BK, 1, true>(P, accs[0], accs[1], ke - kb, smem_base, bar_base, lane, s, ph);
            else if (P.nprod == 3) tile_mainloop<BN, BK, 3, false>(P, accs[0], accs[1], ke - kb, smem_base, bar_base, lane, s, ph);
            else tile_mainloop<BN, BK, 1, false>(P, accs[0], accs[1], ke - kb, smem_base, bar_base, lane, s, ph);
            if (tile == (item + 1) * P.item_tiles - 1 && other_item < total_items)
                asm volatile("bar.arrive %0, 256;" ::"r"(4 - g) : "memory");     // the other warpgroup's next item may start
            if (P.tma_store) {
                store_raw_tma<BN>(P, accs[0], ti, 0, gtid == 0, 1 + g, smem_u32(epi));
                store_raw_tma<BN>(P, accs[1], ti, 1, gtid == 0, 1 + g, smem_u32(epi));
                continue;
            }

            // ---- epilogue (thread = tile row, 16 columns of each 32-column chunk), two 64-row halves
#pragma unroll
            for (int h = 0; h < 2; ++h) {
            float (&acc)[BN / 2] = accs[h];
            float (&racc)[4] = raccs[h];
            const int row = 64 * h + xrow;
            const KParams::Sub& S = P.sub[ti.sub];
            const int tw = row % S.TW, th = (row / S.TW) % S.TH, tnn = row / (S.TW * S.TH);
            const int x = ti.x0 + tw;
            const int n = n0 + tnn;
            const int ox = x * P.ox_mul + S.ox_off;
            const int y = ti.y0 + th;
            const int oy = y * P.oy_mul + S.oy_off;
            const bool valid = !ti.pad && (n < P.N) && (y < S.y_end) && (x < S.x_end) && (oy < P.OH) && (ox < P.OW);
            const int64_t opix = ((int64_t)n * P.OH + oy) * P.OW + ox;
            float nz = 0.f;
            if (valid && P.noise) nz = __ldg(P.noise + (int64_t)n * P.noise_nstride + (int64_t)oy * P.OW + ox);
#pragma unroll 1
            for (int c32 = 0; c32 < BN; c32 += 32) {
                // accumulator columns c32 .. c32+31 -> xbuf[row][column]
                asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
#pragma unroll
                for (int cc = 0; cc < (BN + 31) / 32; ++cc) {
                    if (cc * 32 == c32) {
#pragma unroll
                        for (int e = 0; e < 16; e += 2) {
                            const int i = cc * 16 + e;
                            if (i < BN / 2) {
                                const int r = 16 * (warp & 3) + (lane >> 2) + 8 * ((i >> 1) & 1), c = 8 * ((i >> 2) & 3) + 2 * (lane & 3);
                                *reinterpret_cast<float2*>(xbuf + r * kXStride + c) = make_float2(acc[i], acc[i + 1]);
                            }
                        }
                    }
                }
                asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
                const int c16 = c32 + 16 * half;
                const int co0 = tn * P.block_n + c16;
                if (c16 >= BN || !valid || co0 >= P.Cout) continue;
                uint32_t r[16];
#pragma unroll
                for (int j4 = 0; j4 < 4; ++j4) {
                    const float4 t4 = *reinterpret_cast<const float4*>(xbuf + xrow * kXStride + 16 * half + 4 * j4);
                    r[4 * j4] = __float_as_uint(t4.x); r[4 * j4 + 1] = __float_as_uint(t4.y);
                    r[4 * j4 + 2] = __float_as_uint(t4.z); r[4 * j4 + 3] = __float_as_uint(t4.w);
                }
                const int nco = min(16, P.Cout - co0);
                float v[16], s0[16], s1[16];
                if (staged) {
                    const float4* d4 = reinterpret_cast<const float4*>(stg + c16);
                    const float4* b4 = reinterpret_cast<const float4*>(stg + kMaxBlockN + c16);
                    const float4* p4 = reinterpret_cast<const float4*>(stg + 2 * kMaxBlockN + c16);
                    const float4* q4 = reinterpret_cast<const float4*>(stg + 3 * kMaxBlockN + c16);
#pragma unroll
                    for (int j4 = 0; j4 < 4; ++j4) {
                        const float4 d = d4[j4], bb = b4[j4], ps = p4[j4], qs = q4[j4];
                        const float dd[4] = {d.x, d.y, d.z, d.w}, bv[4] = {bb.x, bb.y, bb.z, bb.w};
                        const float pv[4] = {ps.x, ps.y, ps.z, ps.w}, qv[4] = {qs.x, qs.y, qs.z, qs.w};
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int j = j4 * 4 + e;
                            float a = __uint_as_float(r[j]) * dd[e] + nz + bv[e];
                            a = (a > 0.f ? a : a * P.slope) * P.gain;
                            if (P.clamp >= 0.f) a = fminf(fmaxf(a, -P.clamp), P.clamp);
                            v[j] = a; s0[j] = pv[e]; s1[j] = qv[e];
                        }
                    }
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        if (c < nrgb) {
                            const float4* w4 = reinterpret_cast<const float4*>(stg + (4 + c) * kMaxBlockN + c16);
#pragma unroll
                            for (int j4 = 0; j4 < 4; ++j4) {
                                const float4 w = w4[j4];
                                racc[c] = fmaf(v[j4 * 4], w.x, racc[c]); racc[c] = fmaf(v[j4 * 4 + 1], w.y, racc[c]);
                                racc[c] = fmaf(v[j4 * 4 + 2], w.z, racc[c]); racc[c] = fmaf(v[j4 * 4 + 3], w.w, racc[c]);
                            }
                        }
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        float a = __uint_as_float(r[j]);
                        s0[j] = 1.f; s1[j] = 1.f;
                        if (P.mode == 0 && j < nco) {
                            const int co = co0 + j;
                            if (P.dcoef) a *= __ldg(P.dcoef + (int64_t)n * P.Cout + co);
                            a += nz;
                            if (P.bias) a += __ldg(P.bias + co);
                            a = (a > 0.f ? a : a * P.slope) * P.gain;
                            if (P.clamp >= 0.f) a = fminf(fmaxf(a, -P.clamp), P.clamp);
                            if (P.out[0].style) s0[j] = __ldg(P.out[0].style + (int64_t)n * P.Cout + co);
                            if (P.out[1].style) s1[j] = __ldg(P.out[1].style + (int64_t)n * P.Cout + co);
                        }
                        v[j] = a;
                    }
                }
                // ---- fp32 output (loads of the accumulate path are issued together, before any store, so they overlap)
                if (P.out_f32) {
                    if (P.f32_nchw) {
                        float* dst = P.out_f32 + (((int64_t)n * P.f32_cstride + P.f32_coff + co0) * P.OH + oy) * P.OW + ox;
                        const int64_t cs = (int64_t)P.OH * P.OW;
                        if (P.f32_accumulate) {
                            float old[16];
#pragma unroll
                            for (int j = 0; j < 16; ++j) old[j] = j < nco ? dst[j * cs] : 0.f;
#pragma unroll
                            for (int j = 0; j < 16; ++j) v[j] += old[j];
                        }
#pragma unroll
                        for (int j = 0; j < 16; ++j) if (j < nco) dst[j * cs] = v[j];
                    } else {
                        float* dst = P.out_f32 + (int64_t)ti.split * P.split_stride + opix * P.f32_cstride + P.f32_coff + co0;
                        if (nco == 16 && (((uintptr_t)dst & 31) == 0)) {                 // two full 32-byte sectors per thread
                            if (P.f32_accumulate) {
                                float old[16];
                                ld_global_256(dst, old); ld_global_256(dst + 8, old + 8);
#pragma unroll
                                for (int j = 0; j < 16; ++j) v[j] += old[j];
                            }
                            st_global_256(dst, v); st_global_256(dst + 8, v + 8);
                        } else if (nco == 16 && (((P.f32_cstride | (P.f32_coff + co0)) & 3) == 0)) {
                            if (P.f32_accumulate) {
                                float4 old[4];
#pragma unroll
                                for (int j = 0; j < 4; ++j) old[j] = *reinterpret_cast<const float4*>(dst + 4 * j);
#pragma unroll
                                for (int j = 0; j < 4; ++j) { v[4 * j] += old[j].x; v[4 * j + 1] += old[j].y; v[4 * j + 2] += old[j].z; v[4 * j + 3] += old[j].w; }
                            }
#pragma unroll
                            for (int j = 0; j < 16; j += 4) *reinterpret_cast<float4*>(dst + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
                        } else {
                            if (P.f32_accumulate) {
                                float old[16];
#pragma unroll
                                for (int j = 0; j < 16; ++j) old[j] = j < nco ? dst[j] : 0.f;
#pragma unroll
                                for (int j = 0; j < 16; ++j) v[j] += old[j];
                            }
#pragma unroll
                            for (int j = 0; j < 16; ++j) if (j < nco) dst[j] = v[j];
                        }
                    }
                }
                // ---- split bf16 outputs (next layers' pre-modulated operands), or fp16 single ones in the fp16 instances
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    const N3DSplitOut o = P.out[k];
                    if (!o.hi) continue;
                    if constexpr (F16) {
                        uint32_t h[8];
#pragma unroll
                        for (int j = 0; j < 8; ++j)
                            h[j] = pack_half2(v[2 * j] * (k == 0 ? s0[2 * j] : s1[2 * j]), v[2 * j + 1] * (k == 0 ? s0[2 * j + 1] : s1[2 * j + 1]));
                        __half* dh = (__half*)o.hi + opix * o.cstride + o.coff + co0;
                        if (nco == 16 && (((uintptr_t)dh & 31) == 0)) {
                            st_global_256(dh, h);
                        } else if (nco == 16 && (((o.cstride | (o.coff + co0)) & 7) == 0)) {
#pragma unroll
                            for (int j = 0; j < 8; j += 4) *reinterpret_cast<uint4*>(dh + 2 * j) = make_uint4(h[j], h[j + 1], h[j + 2], h[j + 3]);
                        } else {
#pragma unroll
                            for (int j = 0; j < 16; ++j)
                                if (j < nco) dh[j] = __ushort_as_half((unsigned short)(h[j >> 1] >> ((j & 1) * 16)));
                        }
                    } else {
                        uint32_t h[8], l[8];
#pragma unroll
                        for (int j = 0; j < 8; ++j)
                            split_bf16x2(v[2 * j] * (k == 0 ? s0[2 * j] : s1[2 * j]), v[2 * j + 1] * (k == 0 ? s0[2 * j + 1] : s1[2 * j + 1]), h[j], l[j]);
                        __nv_bfloat16* dh = (__nv_bfloat16*)o.hi + opix * o.cstride + o.coff + co0;
                        __nv_bfloat16* dl = (__nv_bfloat16*)o.lo + opix * o.cstride + o.coff + co0;
                        if (nco == 16 && ((((uintptr_t)dh | (uintptr_t)dl) & 31) == 0)) {           // one full 32-byte sector per array
                            st_global_256(dh, h); st_global_256(dl, l);
                        } else if (nco == 16 && (((o.cstride | (o.coff + co0)) & 7) == 0)) {
#pragma unroll
                            for (int j = 0; j < 8; j += 4) {
                                *reinterpret_cast<uint4*>(dh + 2 * j) = make_uint4(h[j], h[j + 1], h[j + 2], h[j + 3]);
                                *reinterpret_cast<uint4*>(dl + 2 * j) = make_uint4(l[j], l[j + 1], l[j + 2], l[j + 3]);
                            }
                        } else {
#pragma unroll
                            for (int j = 0; j < 16; ++j)
                                if (j < nco) {
                                    dh[j] = __ushort_as_bfloat16((unsigned short)(h[j >> 1] >> ((j & 1) * 16)));
                                    dl[j] = __ushort_as_bfloat16((unsigned short)(l[j >> 1] >> ((j & 1) * 16)));
                                }
                        }
                    }
                }
            }
            if (nrgb > 0 && tile == (item + 1) * P.item_tiles - 1) {     // last n-tile: the two column halves of a row meet in rbuf
                if (half == 1 && valid) *reinterpret_cast<float4*>(rbuf + 4 * xrow) = make_float4(racc[0], racc[1], racc[2], racc[3]);
                asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
                if (half == 0 && valid) {                  // ToRGBLayer: linear bias (+ clamp), added to the up-sampled skip image
                    const float4 o4 = *reinterpret_cast<const float4*>(rbuf + 4 * xrow);
                    const float other[4] = {o4.x, o4.y, o4.z, o4.w};
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        if (c < nrgb) {
                            float o = racc[c] + (BN > 16 ? other[c] : 0.f) + __ldg(P.rgb.bias + c);
                            if (P.rgb.clamp >= 0.f) o = fminf(fmaxf(o, -P.rgb.clamp), P.rgb.clamp);
                            float* dst = P.rgb.nchw ? P.rgb.out + (((int64_t)n * nrgb + c) * P.OH + oy) * P.OW + ox : P.rgb.out + opix * nrgb + c;
                            *dst = P.rgb.accumulate ? (*dst + o) : o;
                        }
                    }
                }
#pragma unroll
                for (int c = 0; c < 4; ++c) racc[c] = 0.f;
            }
            }
        }
        if (other_item < total_items) skip_item(other_item);
        item = other_item;
        }
        if (P.tma_store && gtid == 0) bulk_wait_all();         // the store boxes are read and written before the CTA's memory goes
        // Exit barrier of the cluster: the partner may arrive on this CTA's empty barriers until its consumers are done with
        // their last item, so neither CTA exits before the consumers of both get here.  The producer warpgroup takes no part:
        // its threads exit when they are done, and a cluster barrier waits for the threads that have not exited.  (Its CTA
        // lives while the consumers do, and every multicast it issued lands before the partner's consumers get here.)
        if (P.cluster > 1) cluster_sync();
    }
}

template <int BN, int BK>
__global__ void __launch_bounds__(kThreads, 1) conv_gemm_kernel(const __grid_constant__ KParams P) { conv_gemm_body<BN, BK, false>(P); }
template <int BN, int BK>
__global__ void __launch_bounds__(kThreads, 1) conv_gemm_f16_kernel(const __grid_constant__ KParams P) { conv_gemm_body<BN, BK, true>(P); }

// ---------------------------------------------------------------------------------------------- host side
int pow2_ceil(int v) { int p = 1; while (p < v) p <<= 1; return p; }


}  // namespace

namespace {
// Sub-problem: taps [tap_begin, tap_begin + ntaps) of the launch's tap list over the M-space rectangle [y0, y0 + MH) x [x0, x0 + MW),
// written to output pixel (y * oy_mul + oy_off, x * ox_mul + ox_off).
struct SubSpec { int tap_begin, ntaps, y0, x0, MH, MW, oy_off, ox_off; };

// nint: the first nint sub-problems cover the same rectangle and are interleaved (decode_tile); they are the four parity classes
// of a transposed conv, or the one sub-problem of an ordinary conv.
int launch_conv(const N3DConvGemm* p, const N3DConvTap* taps, int ntaps, int nint, int nsub, const SubSpec* specs, void* stream) {
    N3D_CHECK_ARG(p && p->a_hi && p->w_hi, "n3d_conv_gemm: null operand");
    N3D_CHECK_ARG(p->nprod == 1 || p->nprod == 3, "n3d_conv_gemm: nprod must be 1 or 3");
    N3D_CHECK_ARG(p->f16 == 0 || (p->f16 == 1 && p->nprod == 1), "n3d_conv_gemm: f16 must be 0 or 1, and fp16 operands take nprod 1");
    for (int k = 0; k < 2; ++k)
        N3D_CHECK_ARG(!p->out[k].hi || p->out[k].f16 == p->f16, "n3d_conv_gemm: output %d must be %s (out.f16 = %d)", k,
                      p->f16 ? "fp16 single with fp16 operands" : "split bf16 with bf16 operands", p->f16);
    N3D_CHECK_ARG(p->nprod == 1 || (p->a_lo && p->w_lo), "n3d_conv_gemm: nprod 3 needs lo operands");
    N3D_CHECK_ARG(p->Cin >= 8 && p->Cin % 8 == 0, "n3d_conv_gemm: Cin %d must be a multiple of 8 (TMA 16-byte strides)", p->Cin);
    N3D_CHECK_ARG(p->Cout >= 1 && p->N >= 1, "n3d_conv_gemm: bad sizes");
    N3D_CHECK_ARG(((uintptr_t)p->a_hi & 15) == 0 && ((uintptr_t)p->w_hi & 15) == 0, "n3d_conv_gemm: operands must be 16-byte aligned");
    N3D_CHECK_ARG(p->mode == 0 || (p->mode == 1 && p->out_f32), "n3d_conv_gemm: bad mode");
    // the epilogue's vector stores (float4 / uint4 / 256-bit) test strides and offsets, not the base pointers
    N3D_CHECK_ARG(((uintptr_t)p->out_f32 & 15) == 0, "n3d_conv_gemm: out_f32 must be 16-byte aligned");
    for (int k = 0; k < 2; ++k)
        N3D_CHECK_ARG((((uintptr_t)p->out[k].hi | (uintptr_t)p->out[k].lo) & 15) == 0 && (p->f16 || !p->out[k].hi || p->out[k].lo),
                      "n3d_conv_gemm: split output %d (hi / lo) must be 16-byte aligned, and a split bf16 output needs both", k);
    // the accumulating fp32 store adds the old values into the epilogue's registers before the split outputs are formed from them
    N3D_CHECK_ARG(!p->f32_accumulate || (!p->out[0].hi && !p->out[1].hi), "n3d_conv_gemm: f32_accumulate cannot be combined with split outputs");
    const int splits = p->splits > 1 ? p->splits : 1;
    N3D_CHECK_ARG(splits == 1 || (p->mode == 1 && nsub == 1 && !p->f32_nchw && !p->f32_accumulate && p->split_stride > 0 && p->split_stride % 4 == 0),
                  "n3d_conv_gemm: split-K needs mode 1 (raw NHWC fp32 partial sums) and a split stride that is a multiple of 4");
    cudaStream_t st = (cudaStream_t)stream;

    KParams K;
    memset(&K, 0, sizeof(K));
    K.N = p->N; K.Cout = p->Cout;
    K.splits = splits; K.split_stride = p->split_stride;
    N3D_CHECK_ARG(ntaps >= 1 && ntaps <= 9, "n3d_conv_gemm: %d taps", ntaps);
    for (int t = 0; t < ntaps; ++t) {
        N3D_CHECK_ARG(taps[t].wtap >= 0 && taps[t].wtap < p->T, "n3d_conv_gemm: tap weight slab out of range");
        K.taps[t] = taps[t];
    }
    // Each sub-problem gets the tile geometry of its own M-space: TW up to 16 wide, then TH, then TN images; one A box per
    // distinct geometry.
    K.nsub = nsub; K.nint = nint;
    int tiles_m = 0, sub_m[kMaxSubs], box_sub[kMaxBoxes];     // M tiles per sub-problem; first sub-problem of each box
    for (int i = 0; i < nsub; ++i) {
        const SubSpec& sp = specs[i];
        KParams::Sub& S = K.sub[i];
        N3D_CHECK_ARG(sp.ntaps >= 1 && sp.tap_begin >= 0 && sp.tap_begin + sp.ntaps <= ntaps && sp.MH >= 1 && sp.MW >= 1,
                      "n3d_conv_gemm: bad sub-problem %d", i);
        S.tap_begin = sp.tap_begin; S.ntaps = sp.ntaps;
        S.TW = min(16, pow2_ceil(sp.MW));
        S.TH = min(kBlockM / S.TW, pow2_ceil(sp.MH));
        S.TN = kBlockM / (S.TW * S.TH);
        S.box = 0;
        while (S.box < K.nbox && (K.sub[box_sub[S.box]].TW != S.TW || K.sub[box_sub[S.box]].TH != S.TH)) ++S.box;
        if (S.box == K.nbox) { N3D_CHECK_ARG(K.nbox < kMaxBoxes, "n3d_conv_gemm: too many tile shapes"); box_sub[K.nbox++] = i; }
        S.tiles_x = n3d_div_up(sp.MW, S.TW); S.tiles_y = n3d_div_up(sp.MH, S.TH);
        S.y0 = sp.y0; S.x0 = sp.x0; S.y_end = sp.y0 + sp.MH; S.x_end = sp.x0 + sp.MW;
        S.oy_off = sp.oy_off; S.ox_off = sp.ox_off;
        sub_m[i] = S.tiles_x * S.tiles_y * n3d_div_up(p->N, S.TN);
        tiles_m += sub_m[i];
        N3D_CHECK_ARG(i >= nint || (sp.MH == specs[0].MH && sp.MW == specs[0].MW && sp.y0 == specs[0].y0 && sp.x0 == specs[0].x0),
                      "n3d_conv_gemm: interleaved sub-problems must cover the same M-space");
    }
    // block_n: the largest wgmma N used here not exceeding Cout, halved while the launch has fewer than kMinTiles tiles.  Narrow
    // tiles re-fetch the activation tile once per n-tile, so a few wide tiles beat many narrow ones that merely fill more SMs.
    const int cout16 = ((p->Cout + 15) / 16) * 16;
    int bn = 16;
    int item_tiles = 1;
    {
        const int cands[5] = {128, 96, 64, 32, 16};
        for (int i = 0; i < 5; ++i) {
            if (cands[i] > cout16) continue;
            if (cands[i] == 96 && cout16 % 96 != 0) continue;
            bn = cands[i];
            break;
        }
        const int min_tiles = splits > 1 ? kMinTilesSplit : kMinTiles;     // split launches: short K loops, so spread over (nearly) all SMs
        while (bn > 32 && tiles_m * splits * n3d_div_up(p->Cout, bn) < min_tiles) bn = (bn == 96) ? 32 : bn / 2;
        if (p->rgb.out) {                                   // fused ToRGB: one work item covers every output channel of its pixels
            N3D_CHECK_ARG(cout16 <= 256 && cout16 % 16 == 0, "n3d_conv_gemm: fused ToRGB needs Cout <= 256");
            N3D_CHECK_ARG(p->rgb.channels >= 1 && p->rgb.channels <= 4 && p->rgb.weight && p->rgb.style && p->rgb.bias, "n3d_conv_gemm: bad fused ToRGB descriptor");
            N3D_CHECK_ARG(p->mode == 0 && nsub == 1 && K.sub[0].TN == 1, "n3d_conv_gemm: fused ToRGB needs mode 0 and >= 128 output positions per image");
            bn = kMaxBlockN;                                // the narrowest width holding every channel, else 128-wide n-tiles in turn
            for (const int w : {16, 32, 64, 96, 128}) if (w >= cout16) { bn = w; break; }
            item_tiles = n3d_div_up(p->Cout, bn);
        }
    }
    K.block_n = bn;
    K.tiles_n = n3d_div_up(p->Cout, bn);
    K.item_tiles = item_tiles;
    // block_k: 64-channel stages where the ring still holds kMinStages of them, else 32 (same (tap, 16-channel) MMA sequence, so
    // the same accumulation order either way).  A bf16 stage holds the hi and lo tiles of A and B, an fp16 stage one of each.
    const int tiles_per_stage = p->f16 ? 1 : 2;
    const int block_k = (p->Cin % 64 == 32 || kRingBytes / (tiles_per_stage * (kBlockM + bn) * 64 * 2) < kMinStages) ? 32 : 64;
    K.a_bytes = kBlockM * block_k * 2;
    K.b_bytes = bn * block_k * 2;
    K.stage_bytes = tiles_per_stage * (K.a_bytes + K.b_bytes);
    K.stages = min(kMaxStages, kRingBytes / K.stage_bytes);
    K.cin_chunks = n3d_div_up(p->Cin, block_k);
    if (splits > 1) {                                        // every K slice must own at least one step
        const int nsteps = specs[0].ntaps * K.cin_chunks, per = n3d_div_up(nsteps, splits);
        N3D_CHECK_ARG(per * (splits - 1) < nsteps, "n3d_conv_gemm: %d K slices for %d K steps", splits, nsteps);
    }
    K.nprod = p->nprod; K.a_img_stride = p->a_img_mul;
    N3DDeviceState* D = n3d_device_state();
    if (!D) return N3D_ERR_CUDA;
    const int smem = K.stages * K.stage_bytes + 2 * kEpiBytes + 8 * (2 * K.stages) + 1024;
    typedef void (*ConvKernel)(const KParams);
    const ConvKernel kernels[2][2][5] = {
        {{conv_gemm_kernel<16, 32>, conv_gemm_kernel<32, 32>, conv_gemm_kernel<64, 32>, conv_gemm_kernel<96, 32>, conv_gemm_kernel<128, 32>},
         {conv_gemm_kernel<16, 64>, conv_gemm_kernel<32, 64>, conv_gemm_kernel<64, 64>, conv_gemm_kernel<96, 64>, conv_gemm_kernel<128, 64>}},
        {{conv_gemm_f16_kernel<16, 32>, conv_gemm_f16_kernel<32, 32>, conv_gemm_f16_kernel<64, 32>, conv_gemm_f16_kernel<96, 32>, conv_gemm_f16_kernel<128, 32>},
         {conv_gemm_f16_kernel<16, 64>, conv_gemm_f16_kernel<32, 64>, conv_gemm_f16_kernel<64, 64>, conv_gemm_f16_kernel<96, 64>, conv_gemm_f16_kernel<128, 64>}}};
    const int bi = bn == 16 ? 0 : bn == 32 ? 1 : bn == 64 ? 2 : bn == 96 ? 3 : 4;
    const ConvKernel kern = kernels[p->f16][block_k == 64][bi];
    int rc;
    if ((rc = n3d_smem_optin((const void*)kern, 227 * 1024, "n3d_conv_gemm")) != N3D_OK) return rc;
    // Cluster of 2 for the wide tiles (block_n 96 and 128) without split-K, where some sub-problem has two M tiles to pair.  The
    // pair shares each weight tile (one half-box multicast per CTA), so a stage costs each CTA 2 * (128 + block_n / 2) rows of
    // L2 -> shared traffic instead of 2 * (128 + block_n).  The split-K launches and block_n <= 64 gain nothing from pairing on
    // the H100 (DESIGN.md section 6) and stay unclustered.
    int max_m = 0;
    for (int i = 0; i < nsub; ++i) max_m = max(max_m, sub_m[i]);
    const int cl = (splits == 1 && bn >= 96 && max_m >= 2) ? 2 : 1;
    const int slots = cl == 1 ? D->num_sms : n3d_max_clusters((const void*)kern, kThreads, 227 * 1024, cl, "n3d_conv_gemm");
    if (slots <= 0) return N3D_ERR_CUDA;
    K.cluster = cl; K.b_rows = bn / cl;
    {
        for (int i = 0; i < nsub; ++i) K.sub[i].tiles_m = sub_m[i];
        int end = nint * n3d_div_up(sub_m[0], cl) * K.tiles_n;  // the interleaved sub-problems share one tile_end
        for (int i = 0; i < nsub; ++i) {
            if (i >= nint) end += n3d_div_up(sub_m[i], cl) * K.tiles_n;
            K.sub[i].tile_end = end;
        }
    }
    // Interleaved parity classes go to one CTA (cluster) as a unit (same input rows, equal cost per unit) once there are more of
    // their items than CTAs (clusters); with fewer, each item gets its own (a shorter critical path than a 4 + 2 + 2 + 1-tap unit).
    const int units_grouped = n3d_div_up(sub_m[0], cl) * K.tiles_n;
    K.groups = (nint > 1 && nint * units_grouped > slots) ? units_grouped : 0;
    K.total_items = K.sub[nsub - 1].tile_end * splits / item_tiles;
    const int units = K.total_items - K.groups * (nint - 1);
    K.mode = p->mode; K.dcoef = p->dcoef; K.bias = p->bias; K.noise = p->noise; K.noise_nstride = p->noise_nstride;
    K.gain = p->gain; K.slope = p->slope; K.clamp = p->clamp;
    K.out[0] = p->out[0]; K.out[1] = p->out[1];
    K.out_f32 = p->out_f32; K.f32_cstride = p->f32_cstride; K.f32_coff = p->f32_coff; K.f32_nchw = p->f32_nchw;
    K.f32_accumulate = p->f32_accumulate;
    K.rgb = p->rgb;
    K.oy_mul = p->oy_mul; K.ox_mul = p->ox_mul; K.OH = p->OH; K.OW = p->OW;
    K.err_flag = nullptr;       // a protocol timeout traps (the launch fails with an error); no device-side flag is kept

    // A [NI][AH][AW][Cin] and B [T][Cout][Cin], both packed
    const uint64_t adims[4] = {(uint64_t)p->Cin, (uint64_t)p->AW, (uint64_t)p->AH, (uint64_t)p->NI};
    const uint64_t astr[3] = {adims[0] * 2, adims[0] * adims[1] * 2, adims[0] * adims[1] * adims[2] * 2};
    const uint64_t wdims[3] = {(uint64_t)p->Cin, (uint64_t)p->Cout, (uint64_t)p->T};
    const uint64_t wstr[2] = {wdims[0] * 2, wdims[0] * wdims[1] * 2};
    const uint32_t wbox[3] = {(uint32_t)block_k, (uint32_t)K.b_rows, 1u};   // bn / 2 is a multiple of 8: whole swizzle atoms
    const CUtensorMapSwizzle swz = block_k == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    const CUtensorMapDataType bf16 = p->f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;   // operand type
    for (int b = 0; b < K.nbox; ++b) {
        const KParams::Sub& S = K.sub[box_sub[b]];
        const uint32_t abox[4] = {(uint32_t)block_k, (uint32_t)S.TW, (uint32_t)S.TH, (uint32_t)S.TN};
        if ((rc = n3d_encode_tmap(&K.tmA[b][0], bf16, p->a_hi, 4, adims, astr, abox, swz, "n3d_conv_gemm")) != N3D_OK) return rc;
        if (p->nprod == 3 && (rc = n3d_encode_tmap(&K.tmA[b][1], bf16, p->a_lo, 4, adims, astr, abox, swz, "n3d_conv_gemm")) != N3D_OK) return rc;
    }
    if ((rc = n3d_encode_tmap(&K.tmB_hi, bf16, p->w_hi, 3, wdims, wstr, wbox, swz, "n3d_conv_gemm")) != N3D_OK) return rc;
    if (p->nprod == 3 && (rc = n3d_encode_tmap(&K.tmB_lo, bf16, p->w_lo, 3, wdims, wstr, wbox, swz, "n3d_conv_gemm")) != N3D_OK) return rc;

    // Raw fp32 output through TMA stores: mode 1 with nothing else to write, NHWC, not accumulating, 16-byte aligned pixel stride
    // and channel offset, pixels that do not overlap, and at least one output pixel in every sub-problem (a tensor map has no
    // empty dimension).  Every other descriptor keeps the per-thread stores.  Sub-problem i's map covers the output pixels
    // (y * oy_mul + oy_off, x * ox_mul + ox_off) of x < x_end, y < y_end that lie inside OW x OH.
    {
        const int64_t cs = p->f32_cstride;
        bool tma = p->mode == 1 && !p->out[0].hi && !p->out[1].hi && !p->f32_nchw && !p->f32_accumulate && p->oy_mul >= 1 && p->ox_mul >= 1 &&
                   cs % 4 == 0 && p->f32_coff % 4 == 0 && p->f32_coff >= 0 && cs >= p->f32_coff + p->Cout;
        uint64_t cdims[kMaxSubs][5];
        for (int i = 0; i < nsub && tma; ++i) {
            const KParams::Sub& S = K.sub[i];
            const int xd = min(S.x_end, n3d_div_up(p->OW - S.ox_off, p->ox_mul)), yd = min(S.y_end, n3d_div_up(p->OH - S.oy_off, p->oy_mul));
            const uint64_t d[5] = {(uint64_t)p->Cout, (uint64_t)xd, (uint64_t)yd, (uint64_t)p->N, (uint64_t)splits};
            memcpy(cdims[i], d, sizeof(d));
            tma = S.oy_off >= 0 && S.ox_off >= 0 && xd >= 1 && yd >= 1;
        }
        K.tma_store = tma;
        const int bc = min(32, bn);
        for (int i = 0; i < nsub && tma; ++i) {
            const KParams::Sub& S = K.sub[i];
            const uint64_t pix = (uint64_t)cs * 4, cstr[4] = {p->ox_mul * pix, (uint64_t)p->oy_mul * p->OW * pix, (uint64_t)p->OH * p->OW * pix,
                                                               splits > 1 ? (uint64_t)p->split_stride * 4 : (uint64_t)p->N * p->OH * p->OW * pix};
            const uint32_t cbox[5] = {(uint32_t)bc, (uint32_t)S.TW, (uint32_t)(S.TN > 1 ? S.TH : S.TH / 2), (uint32_t)(S.TN > 1 ? S.TN / 2 : 1), 1u};
            const float* base = p->out_f32 + (((int64_t)S.oy_off * p->OW + S.ox_off) * cs + p->f32_coff);
            if ((rc = n3d_encode_tmap(&K.tmC[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, base, 5, cdims[i], cstr, cbox,
                                      bc == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, "n3d_conv_gemm")) != N3D_OK) return rc;
        }
    }

    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    cfg.gridDim = dim3(cl * min(units, slots));
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    if (cl > 1) {
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = cl; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
    }
    cudaLaunchKernelEx(&cfg, kern, K);
    N3D_CHECK_LAUNCH("n3d_conv_gemm");
    return N3D_OK;
}
}  // namespace

extern "C" int n3d_conv_gemm(const N3DConvGemm* p, void* stream) {
    N3D_CHECK_ARG(p, "n3d_conv_gemm: null descriptor");
    N3D_CHECK_ARG(p->ntaps >= 1 && p->ntaps <= 9, "n3d_conv_gemm: ntaps %d", p->ntaps);
    N3D_CHECK_ARG(p->MH >= 1 && p->MW >= 1, "n3d_conv_gemm: bad M-space");
    const SubSpec sp = {0, p->ntaps, 0, 0, p->MH, p->MW, p->oy_off, p->ox_off};
    return launch_conv(p, p->taps, p->ntaps, 1, 1, &sp, stream);
}

// Stride-2 transposed 3x3 convolution (conv_transpose2d(stride 2), conv2d_resample.py:114-127) as ONE launch: the four
// output-parity classes (a, b) -- out[2p+a, 2q+b] = sum_{ky = a mod 2, kx = b mod 2} W[ky,kx] x[p-(ky-a)/2, q-(kx-b)/2] -- over
// p <= H - a, q <= W - b.  Each class's interior p < H, q < W is one of four interleaved sub-problems (4 / 2 / 2 / 1 taps) with the
// tile geometry of an H x W conv; the extra row p = H (a = 0) and column q = W (b = 0) are five thin sub-problems of their own
// (two row strips, two column strips, one corner pixel), so no tile row or column is spent on a single edge row.  Every output
// pixel sees its class's taps in the same order as in a separate launch of that class.  p->MH, p->MW = INPUT height/width; the
// raw fp32 result [(2H+1), (2W+1)] goes to p->out_f32 (mode 1); taps / offsets / OH / OW of the descriptor are ignored and derived here.
extern "C" int n3d_conv_transposed_gemm(const N3DConvGemm* p, void* stream) {
    N3D_CHECK_ARG(p && p->out_f32, "n3d_conv_transposed_gemm: null descriptor / output");
    N3D_CHECK_ARG(p->T == 9, "n3d_conv_transposed_gemm: needs 3x3 weights (T == 9)");
    N3D_CHECK_ARG(p->MH >= 1 && p->MW >= 1, "n3d_conv_transposed_gemm: bad input size");
    N3DConvGemm q = *p;
    q.mode = 1; q.oy_mul = 2; q.ox_mul = 2; q.OH = 2 * p->MH + 1; q.OW = 2 * p->MW + 1; q.a_img_mul = 0;
    const int H = p->MH, W = p->MW;
    N3DConvTap taps[9];
    SubSpec sp[kMaxSubs];
    int nt = 0;
    for (int c = 0; c < 4; ++c) {                       // classes (0,0), (0,1), (1,0), (1,1): interiors
        const int a = c >> 1, b = c & 1;
        sp[c] = {nt, 0, 0, 0, H, W, a, b};
        for (int ky = 0; ky < 3; ++ky)
            for (int kx = 0; kx < 3; ++kx)
                if ((ky - a) % 2 == 0 && (kx - b) % 2 == 0) {
                    N3DConvTap t;
                    t.dy = (int8_t)(-(ky - a) / 2); t.dx = (int8_t)(-(kx - b) / 2); t.img_off = 0; t.wtap = ky * 3 + kx;
                    taps[nt++] = t;
                    ++sp[c].ntaps;
                }
    }
    auto edge = [&](int c, int y0, int x0, int MH, int MW) { return SubSpec{sp[c].tap_begin, sp[c].ntaps, y0, x0, MH, MW, c >> 1, c & 1}; };
    sp[4] = edge(0, H, 0, 1, W);                        // row p = H of classes (0,0) and (0,1)
    sp[5] = edge(1, H, 0, 1, W);
    sp[6] = edge(0, 0, W, H, 1);                        // column q = W of classes (0,0) and (1,0)
    sp[7] = edge(2, 0, W, H, 1);
    sp[8] = edge(0, H, W, 1, 1);                        // corner (H, W) of class (0,0)
    return launch_conv(&q, taps, nt, 4, 9, sp, stream);
}
