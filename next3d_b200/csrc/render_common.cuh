// Device helpers shared by the fused renderer and the point-sampling kernel (both in render_fused.cu): counter RNG,
// torch.linspace arithmetic, the manual shared-memory swizzles matching the TMA / wgmma SWIZZLE_64B / SWIZZLE_128B layouts, MUFU-based
// activations and the decoder-weight staging (fp32 -> bf16 hi/lo B-operand tiles).
#pragma once
#include "common.cuh"
#include "tc_ptx.cuh"

namespace n3d_rc {

constexpr int kFeat = 32;
constexpr int kHidden = 64;
constexpr int kOut = 33;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

__device__ __forceinline__ float hash_uniform(uint64_t seed, uint64_t idx) {
    uint64_t z = seed + idx * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    return (float)(uint32_t)(z >> 40) * (1.0f / 16777216.0f);
}

// torch.linspace(start, end, steps) for float32: symmetric evaluation around the midpoint
__device__ __forceinline__ float linspace_at(float start, float end, int steps, int i) {
    const float step = (end - start) / (float)(steps - 1);
    return i < steps / 2 ? start + step * (float)i : end - step * (float)(steps - 1 - i);
}

__device__ __forceinline__ uint32_t sw64_off(int row, int byte_in_row) {       // 64-byte rows, Swizzle<2,4,3>
    return (uint32_t)(row * 64 + ((((byte_in_row >> 4) ^ ((row >> 1) & 3)) << 4) | (byte_in_row & 15)));
}
__device__ __forceinline__ uint32_t sw128_off(int row, int byte_in_row) {      // 128-byte rows, Swizzle<3,4,3>
    return (uint32_t)(row * 128 + ((((byte_in_row >> 4) ^ (row & 7)) << 4) | (byte_in_row & 15)));
}

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float lg2_approx(float x) {
    float y;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// softplus(x) with x given as y = x * log2(e):  ln2 * max(log2(1 + 2^min(y,126)), y).  For y > 24 the sum rounds to 2^y and the
// result is x exactly as torch's threshold branch; the min/max pair only keeps 2^y finite for absurd inputs.
__device__ __forceinline__ float softplus_from_log2(float y) {
    const float e = ex2_approx(fminf(y, 126.f));
    return kLn2 * fmaxf(lg2_approx(1.f + e), y);
}
__device__ __forceinline__ float softplus_fast(float x) { return softplus_from_log2(x * kLog2e); }
__device__ __forceinline__ float sigmoid_fast(float x) { return rcp_approx(1.f + ex2_approx(-kLog2e * x)); }

// Camera ray of pixel (row, col) of image n (ray_sampler.py:43-63): origin o and unit direction d.  The renderer and the normal
// pass both call this, so a sample's position o + t * d is the same float expression in both kernels.
__device__ __forceinline__ void camera_ray(const N3DRender& P, int n, int row, int col, float (&o)[3], float (&d)[3]) {
    const float inv = 1.f / (float)P.res, half = 0.5f / (float)P.res;
    const float xc = (float)col * inv + half, yc = (float)row * inv + half;
    const float* I = P.intrinsics + n * 9;
    const float fx = __ldg(I), sk = __ldg(I + 1), cx = __ldg(I + 2), fy = __ldg(I + 4), cy = __ldg(I + 5);
    const float xl = (xc - cx + cy * sk / fy - sk * yc / fy) / fx;
    const float yl = (yc - cy) / fy;
    const float* C = P.cam2world + n * 16;
    float wv[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        wv[a] = __ldg(C + a * 4) * xl + __ldg(C + a * 4 + 1) * yl + __ldg(C + a * 4 + 2) + __ldg(C + a * 4 + 3);
        o[a] = __ldg(C + a * 4 + 3);
        wv[a] -= o[a];
    }
    const float nrm = fmaxf(sqrtf(wv[0] * wv[0] + wv[1] * wv[1] + wv[2] * wv[2]), 1e-12f);
#pragma unroll
    for (int a = 0; a < 3; ++a) d[a] = wv[a] / nrm;
}

}  // namespace n3d_rc
