// Op-level kernels behind torch_utils.ops.{bias_act, upfirdn2d, filtered_lrelu}: the forward passes and bias_act's gradients
// (upfirdn2d's gradient is upfirdn2d itself).
// Memory-bound: one pass, 128-bit accesses where the layout allows, grid sized to the SM count.
#include "common.cuh"

template <typename T> struct Vec4;
template <> struct Vec4<float> { typedef float4 type; };
template <> struct Vec4<__half> { typedef uint2 type; };

__device__ __forceinline__ float n3d_act(float v, int act, float alpha) {
    switch (act) {
        case 1: return v;
        case 2: return v > 0.f ? v : 0.f;
        case 3: return v > 0.f ? v : v * alpha;
        case 4: return tanhf(v);
        case 5: return 1.f / (1.f + expf(-v));
        case 6: return v > 0.f ? v : expm1f(v);
        case 7: return v > 0.f ? 1.0507009873554805f * v : 1.0507009873554805f * 1.6732632423543772f * expm1f(v);
        case 8: return v > 20.f ? v : log1pf(expf(v));
        case 9: return v / (1.f + expf(-v));
    }
    return v;
}

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

// 4 elements per thread per iteration; bias index computed per element (step_b may be 1 for channels_last).  vec == 0 (x or y not
// aligned to a 4-element vector, e.g. a view that starts inside its storage): every element goes through the scalar loop.
template <typename T>
__global__ void __launch_bounds__(256) bias_act_kernel(const T* __restrict__ x, const T* __restrict__ b, T* __restrict__ y,
                                                       int64_t numel, int size_b, int step_b, int act, float alpha,
                                                       float gain, float clamp, int vec) {
    typedef typename Vec4<T>::type V;
    const int64_t nvec = vec ? numel >> 2 : 0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += stride) {
        V v = reinterpret_cast<const V*>(x)[i];
        T* e = reinterpret_cast<T*>(&v);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int64_t idx = i * 4 + k;
            float f = to_f<T>(e[k]);
            if (b) f += to_f<T>(b[(idx / step_b) % size_b]);
            f = n3d_act(f, act, alpha) * gain;
            if (clamp >= 0.f) f = fminf(fmaxf(f, -clamp), clamp);
            e[k] = from_f<T>(f);
        }
        reinterpret_cast<V*>(y)[i] = v;
    }
    // tail
    for (int64_t idx = (nvec << 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < numel; idx += stride) {
        float f = to_f<T>(x[idx]);
        if (b) f += to_f<T>(b[(idx / step_b) % size_b]);
        f = n3d_act(f, act, alpha) * gain;
        if (clamp >= 0.f) f = fminf(fmaxf(f, -clamp), clamp);
        y[idx] = from_f<T>(f);
    }
}

extern "C" int n3d_bias_act(const void* x, const void* b, void* y, int dtype, int64_t numel, int size_b, int step_b,
                            int act, float alpha, float gain, float clamp, void* stream) {
    N3D_CHECK_ARG(numel >= 0, "n3d_bias_act: negative numel");
    N3D_CHECK_ARG(act >= 1 && act <= 9, "n3d_bias_act: act %d out of range", act);
    N3D_CHECK_ARG(dtype == N3D_DTYPE_F32 || dtype == N3D_DTYPE_F16, "n3d_bias_act: unsupported dtype %d", dtype);
    N3D_CHECK_ARG(!b || (size_b > 0 && step_b > 0), "n3d_bias_act: bad bias geometry");
    if (numel == 0) return N3D_OK;                 // nothing to launch; an empty tensor's data pointer may be NULL
    N3D_CHECK_ARG(x && y, "n3d_bias_act: null pointer");
    const int grid = n3d_grid((numel + 3) / 4, 256);        // 4 elements per thread
    const uintptr_t vec_align = dtype == N3D_DTYPE_F32 ? 15 : 7;     // float4 / 4 x half
    const int vec = (((uintptr_t)x | (uintptr_t)y) & vec_align) == 0;
    if (dtype == N3D_DTYPE_F32)
        bias_act_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)x, (const float*)b, (float*)y, numel,
                                                                        size_b, step_b, act, alpha, gain, clamp, vec);
    else
        bias_act_kernel<__half><<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)x, (const __half*)b, (__half*)y,
                                                                         numel, size_b, step_b, act, alpha, gain, clamp, vec);
    N3D_CHECK_LAUNCH("n3d_bias_act");
    return N3D_OK;
}

// ---------------------------------------------------------------------------------------------- bias_act gradients
// The reference plugin's grad modes (bias_act.cu:58-146) in fp32 for both storage types.  grad 1: dx = dy * act'(x + b) * gain,
// act' taken from the saved output (yy = yref / gain) or, for swish, from the saved input xref + b.  grad 2: the derivative of
// grad 1 with respect to its saved input, times dyref.  Elements whose saved output lies on or outside +-clamp get 0 (for swish
// the output is recomputed from xref); a missing yref counts as 0, as in the plugin.
__device__ __forceinline__ float n3d_act_grad(float v, float xr, float yr, float dyr, int grad, int act, float alpha, float gain,
                                              float clamp) {
    const float yy = gain != 0.f ? yr / gain : 0.f;
    float y = 0.f;
    switch (act) {
        case 1: y = grad == 1 ? v : 0.f; break;
        case 2: y = grad == 1 ? (yy > 0.f ? v : 0.f) : 0.f; break;
        case 3: y = grad == 1 ? (yy > 0.f ? v : v * alpha) : 0.f; break;
        case 4: y = grad == 1 ? v * (1.f - yy * yy) : v * (1.f - yy * yy) * (-2.f * yy); break;
        case 5: y = grad == 1 ? v * yy * (1.f - yy) : v * yy * (1.f - yy) * (1.f - 2.f * yy); break;
        case 6: y = grad == 1 ? (yy >= 0.f ? v : v * (yy + 1.f)) : (yy >= 0.f ? 0.f : v * (yy + 1.f)); break;
        case 7: {
            const float s = 1.0507009873554805f, sa = 1.0507009873554805f * 1.6732632423543772f;
            y = grad == 1 ? (yy >= 0.f ? v * s : v * (yy + sa)) : (yy >= 0.f ? 0.f : v * (yy + sa));
            break;
        }
        case 8: {
            const float c = expf(-yy);
            y = grad == 1 ? v * (1.f - c) : v * c * (1.f - c);
            break;
        }
        case 9: {
            const float c = expf(xr), d = c + 1.f;
            if (grad == 1) y = xr > 40.f ? v : v * c * (xr + d) / (d * d);
            else y = xr > 40.f ? 0.f : v * c * (xr * (2.f - d) + 2.f * d) / (d * d * d);
            yr = xr < -80.f ? 0.f : xr / (expf(-xr) + 1.f) * gain;
            break;
        }
    }
    y *= gain * dyr;
    if (clamp >= 0.f && !(yr > -clamp && yr < clamp)) y = 0.f;
    return y;
}

template <typename T>
__global__ void __launch_bounds__(256) bias_act_grad_kernel(const T* __restrict__ dy, const T* __restrict__ b, const T* __restrict__ xref,
                                                            const T* __restrict__ yref, const T* __restrict__ dyref, T* __restrict__ dx,
                                                            int64_t numel, int size_b, int step_b, int grad, int act, float alpha,
                                                            float gain, float clamp) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += stride) {
        float xr = xref ? to_f<T>(xref[i]) : 0.f;
        if (b) xr += to_f<T>(b[(i / step_b) % size_b]);
        const float yr = yref ? to_f<T>(yref[i]) : 0.f;
        const float dyr = dyref ? to_f<T>(dyref[i]) : 1.f;
        dx[i] = from_f<T>(n3d_act_grad(to_f<T>(dy[i]), xr, yr, dyr, grad, act, alpha, gain, clamp));
    }
}

extern "C" int n3d_bias_act_grad(const void* dy, const void* b, const void* xref, const void* yref, const void* dyref, void* dx, int dtype,
                                 int64_t numel, int size_b, int step_b, int grad, int act, float alpha, float gain, float clamp,
                                 void* stream) {
    N3D_CHECK_ARG(numel >= 0, "n3d_bias_act_grad: negative numel");
    N3D_CHECK_ARG(act >= 1 && act <= 9, "n3d_bias_act_grad: act %d out of range", act);
    N3D_CHECK_ARG(grad == 1 || (grad == 2 && act >= 4), "n3d_bias_act_grad: grad mode %d is not defined for act %d", grad, act);
    N3D_CHECK_ARG(dtype == N3D_DTYPE_F32 || dtype == N3D_DTYPE_F16, "n3d_bias_act_grad: unsupported dtype %d", dtype);
    if (numel == 0) return N3D_OK;                 // nothing to launch; an empty tensor's data pointer may be NULL
    N3D_CHECK_ARG(dy && dx, "n3d_bias_act_grad: null pointer");
    N3D_CHECK_ARG(!b || (size_b > 0 && step_b > 0), "n3d_bias_act_grad: bad bias geometry");
    N3D_CHECK_ARG(act != 9 || xref, "n3d_bias_act_grad: null xref (swish differentiates from its input)");
    N3D_CHECK_ARG(act == 1 || act == 9 || yref, "n3d_bias_act_grad: null yref (act %d differentiates from its output)", act);
    N3D_CHECK_ARG(grad == 1 || dyref, "n3d_bias_act_grad: null dyref (grad mode 2)");
    const int grid = n3d_grid(numel, 256);
    if (dtype == N3D_DTYPE_F32)
        bias_act_grad_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)dy, (const float*)b, (const float*)xref,
                                                                             (const float*)yref, (const float*)dyref, (float*)dx, numel,
                                                                             size_b, step_b, grad, act, alpha, gain, clamp);
    else
        bias_act_grad_kernel<__half><<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)dy, (const __half*)b, (const __half*)xref,
                                                                              (const __half*)yref, (const __half*)dyref, (__half*)dx, numel,
                                                                              size_b, step_b, grad, act, alpha, gain, clamp);
    N3D_CHECK_LAUNCH("n3d_bias_act_grad");
    return N3D_OK;
}

// ---------------------------------------------------------------------------------------------- upfirdn2d
// Generic gather formulation: out[oy,ox] = sum_{fy,fx} filt[fy,fx] * xin[(oy*down + fy - pad0) / up] where divisible.
// The filter (<= 32x32 taps) sits in shared memory; consecutive threads walk the output's fastest-varying dim.
struct UpfirdnParams {
    int N, C, H, W, outH, outW, fh, fw, upx, upy, downx, downy, padx0, pady0, flip;
    float gain;
    int64_t xs[4], ys[4];
    int w_fastest;   // 1: iterate ox fastest (NCHW), 0: iterate c fastest (channels_last)
};

template <typename T>
__global__ void __launch_bounds__(256) upfirdn2d_kernel(const T* __restrict__ x, const float* __restrict__ f, T* __restrict__ y,
                                                        UpfirdnParams p) {
    extern __shared__ float sf[];
    for (int i = threadIdx.x; i < p.fh * p.fw; i += blockDim.x) {
        // upfirdn2d correlates with the FLIPPED filter unless flip_filter (upfirdn2d.py:200-201): store it so that
        // sf[fy*fw+fx] multiplies padded-input pixel (oy*down+fy, ox*down+fx).
        const int fy = i / p.fw, fx = i % p.fw;
        const int sy = p.flip ? fy : p.fh - 1 - fy, sx = p.flip ? fx : p.fw - 1 - fx;
        sf[i] = f[sy * p.fw + sx] * p.gain;
    }
    __syncthreads();
    const int64_t total = (int64_t)p.N * p.C * p.outH * p.outW;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        int n, c, oy, ox;
        int64_t t = idx;
        if (p.w_fastest) { ox = t % p.outW; t /= p.outW; oy = t % p.outH; t /= p.outH; c = t % p.C; n = (int)(t / p.C); }
        else             { c = t % p.C; t /= p.C; ox = t % p.outW; t /= p.outW; oy = t % p.outH; n = (int)(t / p.outH); }
        const T* xb = x + n * p.xs[0] + c * p.xs[1];
        float acc = 0.f;
        const int by = oy * p.downy - p.pady0, bx = ox * p.downx - p.padx0;
        for (int fy = 0; fy < p.fh; ++fy) {
            const int uy = by + fy;
            if (uy < 0 || uy % p.upy != 0) continue;
            const int iy = uy / p.upy;
            if (iy >= p.H) continue;
            for (int fx = 0; fx < p.fw; ++fx) {
                const int ux = bx + fx;
                if (ux < 0 || ux % p.upx != 0) continue;
                const int ix = ux / p.upx;
                if (ix >= p.W) continue;
                acc += sf[fy * p.fw + fx] * to_f<T>(xb[iy * p.xs[2] + ix * p.xs[3]]);
            }
        }
        y[n * p.ys[0] + c * p.ys[1] + oy * p.ys[2] + ox * p.ys[3]] = from_f<T>(acc);
    }
}

extern "C" int n3d_upfirdn2d(const void* x, const float* f, void* y, int dtype, int N, int C, int H, int W,
                             const int64_t x_strides[4], const int64_t y_strides[4], int fh, int fw, int upx, int upy,
                             int downx, int downy, int padx0, int padx1, int pady0, int pady1, int flip, float gain,
                             int outH, int outW, void* stream) {
    N3D_CHECK_ARG(x && f && y, "n3d_upfirdn2d: null pointer");
    N3D_CHECK_ARG(dtype == N3D_DTYPE_F32 || dtype == N3D_DTYPE_F16, "n3d_upfirdn2d: unsupported dtype %d", dtype);
    N3D_CHECK_ARG(fh >= 1 && fw >= 1 && fh * fw <= 1024, "n3d_upfirdn2d: filter %dx%d not supported", fh, fw);
    N3D_CHECK_ARG(upx >= 1 && upy >= 1 && downx >= 1 && downy >= 1, "n3d_upfirdn2d: bad up/down factors");
    const int eh = (H * upy + pady0 + pady1 - fh + downy) / downy, ew = (W * upx + padx0 + padx1 - fw + downx) / downx;
    N3D_CHECK_ARG(outH == eh && outW == ew && outH >= 1 && outW >= 1, "n3d_upfirdn2d: output size %dx%d, expected %dx%d",
                  outH, outW, eh, ew);
    UpfirdnParams p;
    p.N = N; p.C = C; p.H = H; p.W = W; p.outH = outH; p.outW = outW; p.fh = fh; p.fw = fw; p.upx = upx; p.upy = upy;
    p.downx = downx; p.downy = downy; p.padx0 = padx0; p.pady0 = pady0; p.flip = flip; p.gain = gain;
    for (int i = 0; i < 4; ++i) { p.xs[i] = x_strides[i]; p.ys[i] = y_strides[i]; }
    p.w_fastest = (y_strides[3] == 1) ? 1 : 0;
    const int64_t total = (int64_t)N * C * outH * outW;
    if (total == 0) return N3D_OK;
    const int grid = n3d_grid(total, 256, 16);
    const size_t smem = (size_t)fh * fw * sizeof(float);
    if (dtype == N3D_DTYPE_F32)
        upfirdn2d_kernel<float><<<grid, 256, smem, (cudaStream_t)stream>>>((const float*)x, f, (float*)y, p);
    else
        upfirdn2d_kernel<__half><<<grid, 256, smem, (cudaStream_t)stream>>>((const __half*)x, f, (__half*)y, p);
    N3D_CHECK_LAUNCH("n3d_upfirdn2d");
    return N3D_OK;
}

// ---------------------------------------------------------------------------------------------- filtered_lrelu
// API completeness (never executed by TriPlaneGenerator.synthesis, SURVEY.md N3): two upfirdn passes through a
// caller-provided fp32 scratch with the bias and the lrelu/gain/clamp fused into them.  No __constant__ filter
// state (the reference's global constant buffer is not stream-safe, filtered_lrelu.cu:81-82).
template <typename T>
__global__ void __launch_bounds__(256) flrelu_up_kernel(const T* __restrict__ x, const T* __restrict__ b, const float* __restrict__ fu,
                                                        float* __restrict__ tmp, int N, int C, int H, int W, int fh, int fw, int up,
                                                        int padx0, int pady0, int flip, int upH, int upW, float gain, float slope,
                                                        float clamp) {
    extern __shared__ float sf[];
    for (int i = threadIdx.x; i < fh * fw; i += blockDim.x) {
        const int fy = i / fw, fx = i % fw;
        const int sy = flip ? fy : fh - 1 - fy, sx = flip ? fx : fw - 1 - fx;
        sf[i] = (fu ? fu[sy * fw + sx] : 1.f) * (float)(up * up);     // the identity filter carries the up^2 gain as well
    }
    __syncthreads();
    const int64_t total = (int64_t)N * C * upH * upW;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int ox = idx % upW; int64_t t = idx / upW; const int oy = t % upH; t /= upH; const int c = t % C;
        const T* xb = x + (t * (int64_t)H) * W;   // t == n*C + c
        const float bias = b ? to_f<T>(b[c]) : 0.f;
        float acc = 0.f;
        for (int fy = 0; fy < fh; ++fy) {
            const int uy = oy + fy - pady0;
            if (uy < 0 || uy % up != 0 || uy / up >= H) continue;
            for (int fx = 0; fx < fw; ++fx) {
                const int ux = ox + fx - padx0;
                if (ux < 0 || ux % up != 0 || ux / up >= W) continue;
                acc += sf[fy * fw + fx] * (to_f<T>(xb[(uy / up) * W + ux / up]) + bias);
            }
        }
        acc = (acc > 0.f ? acc : acc * slope) * gain;
        if (clamp >= 0.f) acc = fminf(fmaxf(acc, -clamp), clamp);
        tmp[idx] = acc;
    }
}

template <typename T>
__global__ void __launch_bounds__(256) flrelu_down_kernel(const float* __restrict__ tmp, const float* __restrict__ fd, T* __restrict__ y,
                                                          int NC, int upH, int upW, int fh, int fw, int down, int flip, int outH,
                                                          int outW) {
    extern __shared__ float sf[];
    for (int i = threadIdx.x; i < fh * fw; i += blockDim.x) {
        const int fy = i / fw, fx = i % fw;
        const int sy = flip ? fy : fh - 1 - fy, sx = flip ? fx : fw - 1 - fx;
        sf[i] = fd ? fd[sy * fw + sx] : 1.f;
    }
    __syncthreads();
    const int64_t total = (int64_t)NC * outH * outW;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int ox = idx % outW; int64_t t = idx / outW; const int oy = t % outH; t /= outH;
        const float* tb = tmp + t * (int64_t)upH * upW;
        float acc = 0.f;
        for (int fy = 0; fy < fh; ++fy)
            for (int fx = 0; fx < fw; ++fx) acc += sf[fy * fw + fx] * tb[(oy * down + fy) * upW + ox * down + fx];
        y[idx] = from_f<T>(acc);
    }
}

extern "C" int n3d_filtered_lrelu(const void* x, const float* fu, const float* fd, const void* b, void* y, float* tmp, int dtype,
                                  int N, int C, int H, int W, int fuh, int fuw, int fdh, int fdw, int up, int down,
                                  int padx0, int padx1, int pady0, int pady1, float gain, float slope, float clamp, int flip,
                                  int outH, int outW, void* stream) {
    N3D_CHECK_ARG(x && y && tmp, "n3d_filtered_lrelu: null pointer");
    N3D_CHECK_ARG(dtype == N3D_DTYPE_F32 || dtype == N3D_DTYPE_F16, "n3d_filtered_lrelu: unsupported dtype %d", dtype);
    N3D_CHECK_ARG(up >= 1 && down >= 1 && fuh * fuw <= 1024 && fdh * fdw <= 1024 && fuh >= 1 && fdh >= 1,
                  "n3d_filtered_lrelu: bad filter / factors");
    const int upH = H * up + pady0 + pady1 - fuh + 1, upW = W * up + padx0 + padx1 - fuw + 1;
    N3D_CHECK_ARG(upH >= fdh && upW >= fdw, "n3d_filtered_lrelu: upsampled image smaller than the down filter");
    N3D_CHECK_ARG(outH == (upH - fdh + down) / down && outW == (upW - fdw + down) / down, "n3d_filtered_lrelu: bad output size");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t t1 = (int64_t)N * C * upH * upW, t2 = (int64_t)N * C * outH * outW;
    const int g1 = n3d_grid(t1, 256, 16), g2 = n3d_grid(t2, 256, 16);
    if (dtype == N3D_DTYPE_F32) {
        flrelu_up_kernel<float><<<g1, 256, fuh * fuw * 4, st>>>((const float*)x, (const float*)b, fu, tmp, N, C, H, W, fuh, fuw, up,
                                                                padx0, pady0, flip, upH, upW, gain, slope, clamp);
        flrelu_down_kernel<float><<<g2, 256, fdh * fdw * 4, st>>>(tmp, fd, (float*)y, N * C, upH, upW, fdh, fdw, down, flip, outH, outW);
    } else {
        flrelu_up_kernel<__half><<<g1, 256, fuh * fuw * 4, st>>>((const __half*)x, (const __half*)b, fu, tmp, N, C, H, W, fuh, fuw, up,
                                                                 padx0, pady0, flip, upH, upW, gain, slope, clamp);
        flrelu_down_kernel<__half><<<g2, 256, fdh * fdw * 4, st>>>(tmp, fd, (__half*)y, N * C, upH, upW, fdh, fdw, down, flip, outH, outW);
    }
    N3D_CHECK_LAUNCH("n3d_filtered_lrelu");
    return N3D_OK;
}
