// MappingNetwork + truncation (networks_stylegan2.py:233-268 via triplane_next3d.py:111-115) as ONE kernel: z -> ws [N, num_ws, 512].
// Replaces ~14 eager ATen launches per call (normalisations, three addmm, leaky-relu, repeat, lerp) that the per-frame loops of
// the inference scripts issue; SURVEY.md section 8 row f4.  One CTA per latent, one warp per output feature (coalesced rows of
// the weight matrices, warp-shuffle dot products); the ~3.1 MB of fp32 weights stay L2-resident across the batch.
// Also here: row interpolation out[f] = sum_k B[f,k] * Y[k] used by the frame drivers (latent interpolation, camera smoothing).
#include "common.cuh"

namespace {
constexpr int kZ = 512, kW = 512, kC = 25, kThreads = 512;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float block_sum(float v, float* red) {          // all threads get the total
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = lane < kThreads / 32 ? red[lane] : 0.f;
    t = warp_sum(t);
    __syncthreads();
    return t;
}

__global__ void __launch_bounds__(kThreads) mapping_kernel(const float* __restrict__ z, const float* __restrict__ c, float c_scale,
                                                           const float* __restrict__ we, const float* __restrict__ be, const float* __restrict__ w0,
                                                           const float* __restrict__ b0, const float* __restrict__ w1, const float* __restrict__ b1,
                                                           const float* __restrict__ w_avg, float psi, int cutoff, int num_ws, float* __restrict__ ws) {
    __shared__ __align__(16) float h[kZ + kW];     // [normalised z | normalised embedding]
    __shared__ __align__(16) float h1[kW];
    __shared__ float red[kThreads / 32];
    __shared__ float cc[kC];
    const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // normalize_2nd_moment(z)
    const float zv = __ldg(z + (int64_t)n * kZ + tid);
    const float zs = block_sum(zv * zv, red);
    h[tid] = zv * rsqrtf(zs / (float)kZ + 1e-8f);
    // embed(c): FullyConnectedLayer(25 -> 512), weight gain 1/sqrt(25); then normalize_2nd_moment
    if (tid < kC) cc[tid] = __ldg(c + (int64_t)n * kC + tid) * c_scale;
    __syncthreads();
    float y = 0.f;
#pragma unroll 5
    for (int i = 0; i < kC; ++i) y = fmaf(cc[i], __ldg(we + tid * kC + i), y);
    y = y * 0.2f + __ldg(be + tid);
    const float ys = block_sum(y * y, red);
    h[kZ + tid] = y * rsqrtf(ys / (float)kW + 1e-8f);
    __syncthreads();
    // fc0: 1024 -> 512, lr_mul 0.01 (weight gain 0.01/sqrt(1024), bias gain 0.01), lrelu(0.2) * sqrt(2)
    const float4* h4 = reinterpret_cast<const float4*>(h);
    for (int o = warp; o < kW; o += kThreads / 32) {
        const float4* wr = reinterpret_cast<const float4*>(w0 + (int64_t)o * (kZ + kW));
        float a = 0.f;
#pragma unroll
        for (int i = 0; i < (kZ + kW) / 128; ++i) {
            const float4 wv = __ldg(wr + i * 32 + lane), hv = h4[i * 32 + lane];
            a = fmaf(wv.x, hv.x, a); a = fmaf(wv.y, hv.y, a); a = fmaf(wv.z, hv.z, a); a = fmaf(wv.w, hv.w, a);
        }
        a = warp_sum(a);
        if (lane == 0) {
            float v = a * (0.01f / 32.f) + __ldg(b0 + o) * 0.01f;
            h1[o] = (v > 0.f ? v : 0.2f * v) * 1.4142135623730951f;
        }
    }
    __syncthreads();
    // fc1: 512 -> 512
    const float4* g4 = reinterpret_cast<const float4*>(h1);
    for (int o = warp; o < kW; o += kThreads / 32) {
        const float4* wr = reinterpret_cast<const float4*>(w1 + (int64_t)o * kW);
        float a = 0.f;
#pragma unroll
        for (int i = 0; i < kW / 128; ++i) {
            const float4 wv = __ldg(wr + i * 32 + lane), hv = g4[i * 32 + lane];
            a = fmaf(wv.x, hv.x, a); a = fmaf(wv.y, hv.y, a); a = fmaf(wv.z, hv.z, a); a = fmaf(wv.w, hv.w, a);
        }
        a = warp_sum(a);
        if (lane == 0) {
            float v = a * (0.01f / 22.627416997969522f) + __ldg(b1 + o) * 0.01f;
            h[o] = (v > 0.f ? v : 0.2f * v) * 1.4142135623730951f;     // h[0..511] is free again
        }
    }
    __syncthreads();
    // broadcast to num_ws layers; truncation: w_avg.lerp(w, psi) on the first `cutoff` layers (torch.lerp's two-sided formula)
    const float w = h[tid];
    float wt = w;
    if (psi != 1.f && w_avg) {
        const float a = __ldg(w_avg + tid), d = w - a;
        wt = psi < 0.5f ? a + psi * d : w - d * (1.f - psi);
    }
    for (int l = 0; l < num_ws; ++l) ws[((int64_t)n * num_ws + l) * kW + tid] = (cutoff < 0 || l < cutoff) ? wt : w;
}

__global__ void __launch_bounds__(256) interp_rows_kernel(const float* __restrict__ B, const float* __restrict__ Y, int F, int K, int64_t D,
                                                          float* __restrict__ out) {
    const int64_t total = (int64_t)F * D;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int f = (int)(i / D);
        const int64_t d = i - (int64_t)f * D;
        float a = 0.f;
        for (int k = 0; k < K; ++k) {
            const float b = __ldg(B + (int64_t)f * K + k);
            if (b != 0.f) a = fmaf(b, __ldg(Y + (int64_t)k * D + d), a);
        }
        out[i] = a;
    }
}
}  // namespace

extern "C" int n3d_mapping(const float* z, const float* c, int N, float c_scale, const float* embed_w, const float* embed_b, const float* fc0_w,
                           const float* fc0_b, const float* fc1_w, const float* fc1_b, const float* w_avg, float truncation_psi,
                           int truncation_cutoff, int num_ws, float* ws, void* stream) {
    N3D_CHECK_ARG(z && c && embed_w && embed_b && fc0_w && fc0_b && fc1_w && fc1_b && ws && N >= 1 && num_ws >= 1, "n3d_mapping: bad args");
    N3D_CHECK_ARG(truncation_psi == 1.f || w_avg, "n3d_mapping: truncation needs w_avg");
    N3D_CHECK_ARG((((uintptr_t)fc0_w | (uintptr_t)fc1_w) & 15) == 0, "n3d_mapping: fc0_w and fc1_w must be 16-byte aligned");   // float4 loads
    mapping_kernel<<<N, kThreads, 0, (cudaStream_t)stream>>>(z, c, c_scale, embed_w, embed_b, fc0_w, fc0_b, fc1_w, fc1_b, w_avg, truncation_psi,
                                                             truncation_cutoff, num_ws, ws);
    N3D_CHECK_LAUNCH("n3d_mapping");
    return N3D_OK;
}

extern "C" int n3d_interp_rows(const float* B, const float* Y, int F, int K, int64_t D, float* out, void* stream) {
    N3D_CHECK_ARG(B && Y && out && F >= 1 && K >= 1 && D >= 1, "n3d_interp_rows: bad args");
    interp_rows_kernel<<<n3d_grid((int64_t)F * D, 256), 256, 0, (cudaStream_t)stream>>>(B, Y, F, K, D, out);
    N3D_CHECK_LAUNCH("n3d_interp_rows");
    return N3D_OK;
}
