// Shared helpers for libnext3d_b200.so (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/next3d_b200.h"       // status codes N3D_OK / N3D_ERR_* of every extern "C" entry point

void n3d_set_error(const char* fmt, ...);

#define N3D_CHECK_ARG(cond, ...)                        \
    do {                                                \
        if (!(cond)) {                                  \
            n3d_set_error(__VA_ARGS__);                 \
            return N3D_ERR_INVALID_ARG;                 \
        }                                               \
    } while (0)

#define N3D_CHECK_LAUNCH(name)                                                       \
    do {                                                                             \
        cudaError_t e__ = cudaGetLastError();                                        \
        if (e__ != cudaSuccess) {                                                    \
            n3d_set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));   \
            return N3D_ERR_CUDA;                                                     \
        }                                                                            \
    } while (0)

static inline int n3d_div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// Host-side facts cached PER DEVICE (the library holds no device memory and no device-global state): SM count, which kernels
// already had their dynamic shared-memory limit raised on that device (n3d_smem_optin), and how many clusters of a kernel fit
// at once (n3d_max_clusters).  Indexed by the current device at call time.
struct N3DDeviceState {
    static constexpr int kSmemSlots = 32;
    int num_sms;
    int n_smem, n_clusters;
    struct { const void* kernel; int bytes; } smem[kSmemSlots];
    struct { const void* kernel; int clusters; } clusters[kSmemSlots];
};
N3DDeviceState* n3d_device_state(void);      // api.cu; nullptr (+ error message) when the current device cannot be queried

// Raises `kernel`'s dynamic shared-memory limit to at least `bytes` on the current device, once per (device, kernel).
// N3D_OK, or N3D_ERR_CUDA with a message that starts with `who`.
int n3d_smem_optin(const void* kernel, int bytes, const char* who);     // api.cu

// TMA descriptor of a tensor of `dtype` elements: `rank` <= 5 dims (innermost first), byte strides of dims 1 .. rank-1, a box of
// `box` elements per dim, `swizzle` shared-memory layout; loads outside the tensor are zero-filled, stores outside it are skipped.
// N3D_OK, or N3D_ERR_CUDA with a message that starts with `who`.
int n3d_encode_tmap(CUtensorMap* tm, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                    const uint32_t* box, CUtensorMapSwizzle swizzle, const char* who);     // api.cu

// Clusters of `cluster` CTAs (`threads` threads, `smem_bytes` dynamic shared memory each) of `kernel` that the current device
// runs at once (cudaOccupancyMaxActiveClusters), queried once per (device, kernel): the kernel's occupancy must not depend on
// the shared memory below `smem_bytes`.  0 with a message that starts with `who` when the query fails.
int n3d_max_clusters(const void* kernel, int threads, int smem_bytes, int cluster, const char* who);     // api.cu

// Grid of a grid-stride launch: one block per `threads` work items, at least 1 and at most `per_sm` blocks per SM of the current
// device.  0 when the device cannot be queried, so that the launch fails and N3D_CHECK_LAUNCH reports it.
inline int n3d_grid(int64_t work_items, int threads, int per_sm = 8) {
    const N3DDeviceState* D = n3d_device_state();
    if (!D) return 0;
    const int64_t g = (work_items + threads - 1) / threads, cap = (int64_t)D->num_sms * per_sm;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// fp32 -> (hi, lo) bf16 pair with hi + lo ~= x to ~16 mantissa bits (used by the 3-product tensor-core scheme).
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(x);
    lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

// Two values at once -> packed bf16x2 words (element a in the low half): one cvt.rn.bf16x2.f32 per word instead of two scalar
// conversions plus a byte permute.  Bit-identical to split_bf16 on each element.
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    const float rx = __fadd_rn(a, -__uint_as_float(hi << 16)), ry = __fadd_rn(b, -__uint_as_float(hi & 0xffff0000u));   // exact
    const __nv_bfloat162 l = __floats2bfloat162_rn(rx, ry);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

// Two values -> one packed fp16x2 word (element a in the low half), each rounded to nearest: the fp16 single form.
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

// 32-byte global accesses as two 128-bit halves (sm_90 has no 256-bit LDG/STG): both halves of one sector per thread and call.
// `p` must be 32-byte aligned.
__device__ __forceinline__ void st_global_256(void* p, const uint32_t (&w)[8]) {
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(w[0], w[1], w[2], w[3]);
    q[1] = make_uint4(w[4], w[5], w[6], w[7]);
}
__device__ __forceinline__ void st_global_256(float* p, const float* v) {
    float4* q = reinterpret_cast<float4*>(p);
    q[0] = make_float4(v[0], v[1], v[2], v[3]);
    q[1] = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void ld_global_256(const float* p, float* v) {
    const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

// read-only variant (non-coherent path)
__device__ __forceinline__ void ldg_nc_256(const float* p, float* v) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b) {
    return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}
