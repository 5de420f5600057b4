// sm_90a PTX wrappers shared by the tensor-core kernels: mbarrier, TMA bulk-tensor loads, wgmma shared-memory descriptors and
// warpgroup MMAs (accumulator in registers), warp-level mma.sync, proxy fences.  The descriptor bit layout follows
// cute::GMMA::GmmaDescriptor.
#pragma once
#include <cuda.h>
#include <stdint.h>

namespace n3d_tc {

constexpr uint32_t kSpinLimit = 1u << 24;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster (which may be this CTA).  Default (CTA
// scope) release, as for a local arrive: it only signals that this thread's reads of a stage are done (their wgmmas retired).
// A .cluster-scope release would compile to a GPU-wide memory barrier per arrive, which waits for the epilogue's global stores.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t rank) {
    asm volatile(
        "{\n\t.reg .b32 remote;\n\t"
        "mapa.shared::cluster.u32 remote, %0, %1;\n\t"
        "mbarrier.arrive.shared::cluster.b64 _, [remote];\n\t}"
        ::"r"(bar), "r"(rank) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// cluster index and number of clusters along x (blockIdx.x and gridDim.x for a launch without clusters)
__device__ __forceinline__ int cluster_idx_x() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
    return (int)r;
}
__device__ __forceinline__ int num_clusters_x() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r));
    return (int)r;
}
// Cluster barrier: arrive (release), then wait (acquire) for every thread of the cluster that has not exited.  Not .aligned:
// warps may be diverged here.
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug traps (kernel aborts with an error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int* err_flag, int code) {
#pragma unroll 1
    for (uint32_t it = 0; it < kSpinLimit; ++it)
        if (mbar_try_wait(bar, parity)) return;
    if (err_flag) atomicExch(err_flag, code);
    __trap();
}

// try_wait with a suspend-time hint: the thread sleeps in hardware until the phase completes (or the hint expires) instead of
// burning issue slots in a polling loop.  Still bounded: a protocol bug traps.
__device__ __forceinline__ void mbar_wait_sleep(uint32_t bar, uint32_t parity, unsigned backoff_ns = 0) {
#pragma unroll 1
    for (uint32_t it = 0; it < (1u << 20); ++it) {
        uint32_t ok;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(bar), "r"(parity), "r"(0x989680u) : "memory");
        if (ok) return;
        if (backoff_ns) __nanosleep(backoff_ns);
    }
    __trap();
}

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// 3-D tensor load multicast to the CTAs of `cta_mask`: the box lands at shared offset `dst` of each of them and signals the
// mbarrier at offset `bar` of each.
__device__ __forceinline__ void tma_load_3d_multicast(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, int c2, uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5}], [%2], %6;"
        ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "h"(cta_mask) : "memory");
}
// 1-D bulk copy global -> shared (TMA engine, no tensor map): `bytes` contiguous bytes, 16-byte aligned on both sides, completion
// counted on the mbarrier like the tensor loads.
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// Suspended wait with a short hint (20 us per try) for kernels whose stages complete within microseconds; bounded (a protocol bug
// traps after about a minute instead of hanging; generous enough for profiler replays and time-sliced contexts).
__device__ __forceinline__ void mbar_wait_short(uint32_t bar, uint32_t parity) {
#pragma unroll 1
    for (uint32_t it = 0; it < (1u << 22); ++it) {
        uint32_t ok;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(bar), "r"(parity), "r"(20000u) : "memory");
        if (ok) return;
    }
    __trap();
}
// 5-D tensor store shared -> global (TMA engine), tracked by the issuing thread's bulk async-groups: the box at `src` (laid out
// and swizzled as the tensor map's box) is written to the tensor at the given coordinates; elements outside the tensor are
// skipped.  The thread that issued it commits the group and later waits for it.
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* tm, uint32_t src, int c0, int c1, int c2, int c3, int c4) {
    asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
                 ::"l"(tm), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every committed group of this thread has finished reading its shared-memory source (its global writes may still be in flight)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// every committed group of this thread is complete
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory");
}

// K-major swizzled shared-memory matrix descriptor (cute::GMMA::GmmaDescriptor): start>>4 [0,14), LBO>>4 [16,30) (unused for
// swizzled K-major, 1), SBO>>4 [32,46) = bytes between 8-row groups, layout [62,64): SWIZZLE_128B = 1, SWIZZLE_64B = 2.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint64_t hi_bits) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | hi_bits;
}
// hi bits for a tile whose rows are block_k bf16 wide: 64 -> 128-byte rows, SWIZZLE_128B; 32 -> 64-byte rows, SWIZZLE_64B
__device__ __forceinline__ constexpr uint64_t wgmma_desc_hi(int block_k) {
    return block_k == 64 ? (((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62)) : (((uint64_t)(512 >> 4) << 32) | ((uint64_t)2 << 62));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int Pending>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(Pending) : "memory"); }

// D[64 x N] (+)= A[64 x 16] * B[16 x N]^T, bf16 (wgmma_bf16) or fp16 (wgmma_f16) operands from shared memory (both K-major), fp32
// accumulator in registers (d[i]: row 16 * (warp % 4) + lane / 4 + 8 * ((i / 2) % 2), column 8 * (i / 4) + 2 * (lane % 4) + i % 2).
// scale_d = 0 overwrites.  N3D_WGMMA_<N>(TY) is the instruction for operand type TY ("bf16" or "f16").
#define N3D_WGMMA_16(TY) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n16k16.f32." TY "." TY " {" \
        "%0, %1, %2, %3, %4, %5, %6, %7" \
        "}, %8, %9, p, 1, 1, 0, 0;\n\t}" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]) \
        : "l"(da), "l"(db), "r"(scale_d));
#define N3D_WGMMA_32(TY) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n32k16.f32." TY "." TY " {" \
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15" \
        "}, %16, %17, p, 1, 1, 0, 0;\n\t}" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]) \
        : "l"(da), "l"(db), "r"(scale_d));
#define N3D_WGMMA_64(TY) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " {" \
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31" \
        "}, %32, %33, p, 1, 1, 0, 0;\n\t}" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
        : "l"(da), "l"(db), "r"(scale_d));
#define N3D_WGMMA_96(TY) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n96k16.f32." TY "." TY " {" \
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47" \
        "}, %48, %49, p, 1, 1, 0, 0;\n\t}" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]) \
        : "l"(da), "l"(db), "r"(scale_d));
#define N3D_WGMMA_128(TY) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " {" \
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63" \
        "}, %64, %65, p, 1, 1, 0, 0;\n\t}" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
        : "l"(da), "l"(db), "r"(scale_d));
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_bf16<16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) { N3D_WGMMA_16("bf16"); }
template <> __device__ __forceinline__ void wgmma_f16<16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) { N3D_WGMMA_16("f16"); }
template <> __device__ __forceinline__ void wgmma_bf16<32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) { N3D_WGMMA_32("bf16"); }
template <> __device__ __forceinline__ void wgmma_f16<32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) { N3D_WGMMA_32("f16"); }
template <> __device__ __forceinline__ void wgmma_bf16<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) { N3D_WGMMA_64("bf16"); }
template <> __device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) { N3D_WGMMA_64("f16"); }
template <> __device__ __forceinline__ void wgmma_bf16<96>(float (&d)[48], uint64_t da, uint64_t db, uint32_t scale_d) { N3D_WGMMA_96("bf16"); }
template <> __device__ __forceinline__ void wgmma_f16<96>(float (&d)[48], uint64_t da, uint64_t db, uint32_t scale_d) { N3D_WGMMA_96("f16"); }
template <> __device__ __forceinline__ void wgmma_bf16<128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) { N3D_WGMMA_128("bf16"); }
template <> __device__ __forceinline__ void wgmma_f16<128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) { N3D_WGMMA_128("f16"); }
template <int N, bool F16>
__device__ __forceinline__ void wgmma_k16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
    if constexpr (F16) wgmma_f16<N>(d, da, db, scale_d);
    else wgmma_bf16<N>(d, da, db, scale_d);
}
// One pipeline stage of a 128-row tile's MMAs (conv_gemm_kernel and conv_wgrad_kernel) as a fixed instruction sequence: one fence,
// BK/16 x NPROD x 2 wgmmas back to back, one commit.  The warpgroup owns all 128 rows of the A tile: acc0 = rows 0-63, acc1 = rows
// 64-127 (two m64 wgmmas sharing the B descriptor).  Per k16 step the products are hi*hi, then (NPROD == 3) hi*lo and lo*hi, so
// every kernel that runs this stage sums in the same order.  FIRST (the first stage of a tile) overwrites the accumulator with its
// first product instead of adding to it.  F16: fp16 operands (NPROD 1; the lo addresses are not read).
template <int BN, int BK, int NPROD, bool FIRST, bool F16 = false>
__device__ __forceinline__ void stage_mma(float (&acc0)[BN / 2], float (&acc1)[BN / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo) {
    constexpr uint32_t h1 = 64u * BK * 2u;         // rows 64-127 of the A tile
    constexpr uint64_t dhi = wgmma_desc_hi(BK);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
        const uint32_t koff = (uint32_t)k * 32u;     // 16 bf16 = 32 bytes inside the swizzle row
        wgmma_k16<BN, F16>(acc0, wgmma_desc(a_hi + koff, dhi), wgmma_desc(b_hi + koff, dhi), (FIRST && k == 0) ? 0u : 1u);
        wgmma_k16<BN, F16>(acc1, wgmma_desc(a_hi + h1 + koff, dhi), wgmma_desc(b_hi + koff, dhi), (FIRST && k == 0) ? 0u : 1u);
        if (NPROD == 3 && !F16) {
            wgmma_bf16<BN>(acc0, wgmma_desc(a_hi + koff, dhi), wgmma_desc(b_lo + koff, dhi), 1u);
            wgmma_bf16<BN>(acc1, wgmma_desc(a_hi + h1 + koff, dhi), wgmma_desc(b_lo + koff, dhi), 1u);
            wgmma_bf16<BN>(acc0, wgmma_desc(a_lo + koff, dhi), wgmma_desc(b_hi + koff, dhi), 1u);
            wgmma_bf16<BN>(acc1, wgmma_desc(a_lo + h1 + koff, dhi), wgmma_desc(b_hi + koff, dhi), 1u);
        }
    }
    wgmma_commit();
}

// warp-level D[16 x 8] += A[16 x 16] * B[16 x 8], bf16 operands in registers (PTX fragment layouts of mma.m16n8k16), fp32 accumulate
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// generic-proxy shared-memory writes (st.shared) -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

}  // namespace n3d_tc
