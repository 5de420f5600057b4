// Vertex colours of a head mesh from rendered views (next3d_b200/bake.py; DESIGN.md section 3.8): the voxel -> world map of the
// shape grid, a z-buffer of the mesh in every view, and a per-vertex blend of the views.  Every floating-point operation is an
// explicitly rounded fp32 intrinsic (no contraction into FMA), so tests/bake_oracle.py restates the results bit for bit in numpy.
#include "common.cuh"

namespace {

__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float dvd(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float lerp(float a, float b, float t) { return add(a, mul(sub(b, a), t)); }

constexpr int kThreads = 256;
constexpr int kSmallBox = 32;          // triangles whose clipped box holds more pixels are rasterised by the whole warp

// World point of a vertex (x, y, z) = (a2, a1, a0) of the flipped grid of create_samples(R, cube): the reference divides the flat
// index in float, so the columns are sheared: s2 = x, s1 = y + x / R, s0 = (R - 1 - z) + s1 / R, and p = s * vs - cube / 2.
__device__ __forceinline__ void voxel_to_world(float x, float y, float z, int R, float cube, float (&p)[3]) {
    const float inv = dvd(1.f, (float)R), vs = dvd(cube, (float)(R - 1)), h = mul(cube, 0.5f);
    const float s1 = add(y, mul(x, inv));
    const float s0 = add(sub((float)(R - 1), z), mul(s1, inv));
    p[0] = sub(mul(s0, vs), h);
    p[1] = sub(mul(s1, vs), h);
    p[2] = sub(mul(x, vs), h);
}

// Projection of world point p into view v: camera depth z (along the camera's +z axis) and continuous pixel coordinates (u, w)
// with pixel centres at integers, the inverse of the renderer's camera_ray (render_common.cuh).
struct Proj {
    float u, w, z;
};
__device__ __forceinline__ Proj project(const float* C, const float* I, const float (&p)[3], int H, int W) {
    const float d0 = sub(p[0], __ldg(C + 3)), d1 = sub(p[1], __ldg(C + 7)), d2 = sub(p[2], __ldg(C + 11));
    float q[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) q[j] = add(add(mul(__ldg(C + j), d0), mul(__ldg(C + 4 + j), d1)), mul(__ldg(C + 8 + j), d2));
    const float xl = dvd(q[0], q[2]), yl = dvd(q[1], q[2]);
    const float xc = add(add(mul(__ldg(I), xl), mul(__ldg(I + 1), yl)), __ldg(I + 2));
    const float yc = add(mul(__ldg(I + 4), yl), __ldg(I + 5));
    return {sub(mul(xc, (float)W), 0.5f), sub(mul(yc, (float)H), 0.5f), q[2]};
}

// A triangle projected into one view: pixel-space corners, reciprocal depths, signed area, clipped pixel box.
struct Tri {
    float u[3], w[3], iz[3], area;
    int c0, c1, r0, r1;
    uint32_t id;
};

__device__ __forceinline__ bool setup(const float* verts, int64_t nv, const int32_t* faces, int64_t f, const float* C, const float* I,
                                      int H, int W, float near, Tri& t) {
    t.id = (uint32_t)f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int32_t i = faces[3 * f + k];
        if (i < 0 || i >= nv) return false;
        const float p[3] = {verts[3 * (int64_t)i], verts[3 * (int64_t)i + 1], verts[3 * (int64_t)i + 2]};
        const Proj q = project(C, I, p, H, W);
        if (!(q.z > near) || !isfinite(q.u) || !isfinite(q.w)) return false;          // at or behind the near plane
        t.u[k] = q.u;
        t.w[k] = q.w;
        t.iz[k] = dvd(1.f, q.z);
    }
    t.area = sub(mul(sub(t.u[1], t.u[0]), sub(t.w[2], t.w[0])), mul(sub(t.w[1], t.w[0]), sub(t.u[2], t.u[0])));
    if (!(t.area != 0.f) || !isfinite(t.area)) return false;                          // degenerate (or overflowing) triangle
    const float umin = fminf(fminf(t.u[0], t.u[1]), t.u[2]), umax = fmaxf(fmaxf(t.u[0], t.u[1]), t.u[2]);
    const float wmin = fminf(fminf(t.w[0], t.w[1]), t.w[2]), wmax = fmaxf(fmaxf(t.w[0], t.w[1]), t.w[2]);
    t.c0 = (int)fminf(fmaxf(ceilf(umin), 0.f), (float)W);
    t.c1 = (int)fminf(fmaxf(floorf(umax), -1.f), (float)(W - 1));
    t.r0 = (int)fminf(fmaxf(ceilf(wmin), 0.f), (float)H);
    t.r1 = (int)fminf(fmaxf(floorf(wmax), -1.f), (float)(H - 1));
    return t.c0 <= t.c1 && t.r0 <= t.r1;
}

// Edge function of pixel centre (px, py) against edge a -> b.
__device__ __forceinline__ float edge(float ua, float wa, float ub, float wb, float px, float py) {
    return sub(mul(sub(ub, ua), sub(py, wa)), mul(sub(wb, wa), sub(px, ua)));
}

// Covers pixel (row, col) with the triangle if its centre is inside or on an edge: key = (depth bits << 32) | triangle id, depth
// the perspective-correct camera depth 1 / sum(b_k / z_k).  Depths are positive, so their bits order as the values do.
__device__ __forceinline__ void cover(const Tri& t, int row, int col, unsigned long long* zb, int W) {
    const float px = (float)col, py = (float)row;
    float e0 = edge(t.u[1], t.w[1], t.u[2], t.w[2], px, py);
    float e1 = edge(t.u[2], t.w[2], t.u[0], t.w[0], px, py);
    float e2 = edge(t.u[0], t.w[0], t.u[1], t.w[1], px, py);
    float area = t.area;
    if (area < 0.f) {
        e0 = -e0;
        e1 = -e1;
        e2 = -e2;
        area = -area;
    }
    if (e0 < 0.f || e1 < 0.f || e2 < 0.f) return;
    const float iz = add(add(mul(dvd(e0, area), t.iz[0]), mul(dvd(e1, area), t.iz[1])), mul(dvd(e2, area), t.iz[2]));
    const float z = dvd(1.f, iz);
    const unsigned long long key = ((unsigned long long)__float_as_uint(z) << 32) | t.id;
    atomicMin(zb + (int64_t)row * W + col, key);
}

// One thread per (view, triangle), view-major.  A thread loops over its triangle's clipped box; a triangle whose box holds more
// than kSmallBox pixels is instead rasterised by its whole warp, 32 pixels at a time, after the small ones.
__global__ void __launch_bounds__(kThreads) zbuffer_kernel(const float* __restrict__ verts, int64_t nv, const int32_t* __restrict__ faces,
                                                           int64_t nf, const float* __restrict__ cam2world, const float* __restrict__ intr,
                                                           int views, int H, int W, float near, unsigned long long* __restrict__ zbuf) {
    const int64_t total = nf * views, stride = (int64_t)gridDim.x * blockDim.x;
    const int lane = threadIdx.x & 31;
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < total; base += stride) {
        const int64_t g = base + threadIdx.x;
        Tri t;
        bool ok = false;
        int v = 0;
        if (g < total) {
            v = (int)(g / nf);
            ok = setup(verts, nv, faces, g - (int64_t)v * nf, cam2world + 16 * v, intr + 9 * v, H, W, near, t);
        }
        unsigned long long* zb = zbuf + (int64_t)v * H * W;
        const int64_t box = ok ? (int64_t)(t.c1 - t.c0 + 1) * (t.r1 - t.r0 + 1) : 0;
        if (ok && box <= kSmallBox) {
            for (int r = t.r0; r <= t.r1; ++r)
                for (int c = t.c0; c <= t.c1; ++c) cover(t, r, c, zb, W);
        }
        unsigned big = __ballot_sync(0xffffffffu, box > kSmallBox);
        while (big) {
            const int src = __ffs(big) - 1;
            big &= big - 1;
            Tri s;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                s.u[k] = __shfl_sync(0xffffffffu, t.u[k], src);
                s.w[k] = __shfl_sync(0xffffffffu, t.w[k], src);
                s.iz[k] = __shfl_sync(0xffffffffu, t.iz[k], src);
            }
            s.area = __shfl_sync(0xffffffffu, t.area, src);
            s.c0 = __shfl_sync(0xffffffffu, t.c0, src);
            s.c1 = __shfl_sync(0xffffffffu, t.c1, src);
            s.r0 = __shfl_sync(0xffffffffu, t.r0, src);
            s.r1 = __shfl_sync(0xffffffffu, t.r1, src);
            s.id = __shfl_sync(0xffffffffu, t.id, src);
            const int sv = __shfl_sync(0xffffffffu, v, src);
            const int bw = s.c1 - s.c0 + 1;
            const int64_t n = (int64_t)bw * (s.r1 - s.r0 + 1);
            for (int64_t k = lane; k < n; k += 32) cover(s, s.r0 + (int)(k / bw), s.c0 + (int)(k % bw), zbuf + (int64_t)sv * H * W, W);
        }
    }
}

__global__ void __launch_bounds__(kThreads) world_kernel(const float* __restrict__ verts, int64_t nv, int R, float cube,
                                                         float* __restrict__ world) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x) {
        float p[3];
        voxel_to_world(verts[3 * i], verts[3 * i + 1], verts[3 * i + 2], R, cube, p);
        world[3 * i] = p[0];
        world[3 * i + 1] = p[1];
        world[3 * i + 2] = p[2];
    }
}

struct Bake {
    const float *verts, *world, *grid;
    int64_t nv;
    int R;
    const float *cam2world, *intr, *images;
    int views, H, W;
    const unsigned long long* zbuf;
    float near, eps;
    const float* fallback;
    int fallback_stride;
    uint8_t* colors;
    uint8_t* visible;
    float* weights;
};

// Central-difference gradient of the grid at node (a0, a1, a2), the neighbours clamped to the grid: (d/dx, d/dy, d/dz) with
// x = a2, y = a1, z = a0.
__device__ __forceinline__ void node_gradient(const float* g, int R, int a0, int a1, int a2, float (&d)[3]) {
    const int64_t R2 = (int64_t)R * R;
    const float* row = g + a0 * R2 + (int64_t)a1 * R;
    d[0] = mul(sub(__ldg(row + min(a2 + 1, R - 1)), __ldg(row + max(a2 - 1, 0))), 0.5f);
    d[1] = mul(sub(__ldg(g + a0 * R2 + (int64_t)min(a1 + 1, R - 1) * R + a2), __ldg(g + a0 * R2 + (int64_t)max(a1 - 1, 0) * R + a2)), 0.5f);
    d[2] = mul(sub(__ldg(g + min(a0 + 1, R - 1) * R2 + (int64_t)a1 * R + a2), __ldg(g + max(a0 - 1, 0) * R2 + (int64_t)a1 * R + a2)), 0.5f);
}

// Cell origin and fraction of voxel coordinate c on an axis of R >= 2 nodes.
__device__ __forceinline__ int cell(float c, int R, float& f) {
    const int i = (int)fminf(fmaxf(floorf(c), 0.f), (float)(R - 2));
    f = sub(c, (float)i);
    return i;
}

__global__ void __launch_bounds__(kThreads) bake_kernel(Bake b) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < b.nv; i += (int64_t)gridDim.x * blockDim.x) {
        const float x = b.verts[3 * i], y = b.verts[3 * i + 1], z = b.verts[3 * i + 2];
        const float p[3] = {b.world[3 * i], b.world[3 * i + 1], b.world[3 * i + 2]};
        // trilinear interpolation of the node gradients: along x, then y, then z
        float fx, fy, fz;
        const int i2 = cell(x, b.R, fx), i1 = cell(y, b.R, fy), i0 = cell(z, b.R, fz);
        float gv[3];
        float gz[2][3];
#pragma unroll
        for (int dz = 0; dz < 2; ++dz) {
            float gy[2][3];
#pragma unroll
            for (int dy = 0; dy < 2; ++dy) {
                float g0[3], g1[3];
                node_gradient(b.grid, b.R, i0 + dz, i1 + dy, i2, g0);
                node_gradient(b.grid, b.R, i0 + dz, i1 + dy, i2 + 1, g1);
#pragma unroll
                for (int k = 0; k < 3; ++k) gy[dy][k] = lerp(g0[k], g1[k], fx);
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) gz[dz][k] = lerp(gy[0][k], gy[1][k], fy);
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) gv[k] = lerp(gz[0][k], gz[1][k], fz);
        // outward normal -grad sigma in world space: the map's Jacobian is vs * [[1/R^2, 1/R, -1], [1/R, 1, 0], [1, 0, 0]], whose
        // inverse transpose takes (gx, gy, gz) to (-gz, gy + gz / R, gx - gy / R) up to the factor 1 / vs
        const float inv = dvd(1.f, (float)b.R);
        float n[3] = {gv[2], -add(gv[1], mul(gv[2], inv)), sub(mul(gv[1], inv), gv[0])};
        const float len = __fsqrt_rn(add(add(mul(n[0], n[0]), mul(n[1], n[1])), mul(n[2], n[2])));
        if (len > 0.f) {
#pragma unroll
            for (int k = 0; k < 3; ++k) n[k] = dvd(n[k], len);
        } else {
            n[0] = n[1] = n[2] = 0.f;
        }
        float sw = 0.f, sc[3] = {0.f, 0.f, 0.f};
        for (int v = 0; v < b.views; ++v) {
            const float* C = b.cam2world + 16 * v;
            const Proj q = project(C, b.intr + 9 * v, p, b.H, b.W);
            bool vis = false;
            float w = 0.f;
            if (q.z > b.near) {
                const float cr = floorf(add(q.w, 0.5f)), cc = floorf(add(q.u, 0.5f));
                if (cr >= 0.f && cr < (float)b.H && cc >= 0.f && cc < (float)b.W) {
                    const unsigned long long key = b.zbuf[((int64_t)v * b.H + (int)cr) * b.W + (int)cc];
                    const float zb = key == ~0ull ? __int_as_float(0x7f800000) : __uint_as_float((uint32_t)(key >> 32));
                    vis = q.z <= add(zb, b.eps);
                }
            }
            if (vis) {
                const float e0 = sub(__ldg(C + 3), p[0]), e1 = sub(__ldg(C + 7), p[1]), e2 = sub(__ldg(C + 11), p[2]);
                const float dl = __fsqrt_rn(add(add(mul(e0, e0), mul(e1, e1)), mul(e2, e2)));
                const float c = fmaxf(dvd(add(add(mul(n[0], e0), mul(n[1], e1)), mul(n[2], e2)), dl), 0.f);
                w = mul(c, c);
            }
            if (b.visible) b.visible[(int64_t)v * b.nv + i] = vis;
            if (b.weights) b.weights[(int64_t)v * b.nv + i] = w;
            if (w > 0.f) {
                // bilinear sample, the taps clamped to the image
                const float u0 = floorf(q.u), w0 = floorf(q.w);
                const float tu = sub(q.u, u0), tw = sub(q.w, w0);
                const int ca = min(max((int)u0, 0), b.W - 1), cb = min(max((int)u0 + 1, 0), b.W - 1);
                const int ra = min(max((int)w0, 0), b.H - 1), rb = min(max((int)w0 + 1, 0), b.H - 1);
                sw = add(sw, w);
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const float* im = b.images + ((int64_t)v * 3 + k) * b.H * b.W;
                    const float top = lerp(__ldg(im + (int64_t)ra * b.W + ca), __ldg(im + (int64_t)ra * b.W + cb), tu);
                    const float bot = lerp(__ldg(im + (int64_t)rb * b.W + ca), __ldg(im + (int64_t)rb * b.W + cb), tu);
                    sc[k] = add(sc[k], mul(w, lerp(top, bot, tw)));
                }
            }
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            // no view: the decoder's colour (sigmoid range, as n3d_sample_points writes it), rescaled to the images' -1..1 as the
            // ray marcher rescales its composite (rgb * 2 - 1), so that it shows as image_raw shows it
            const float c = sw > 0.f ? dvd(sc[k], sw) : sub(mul(b.fallback[i * b.fallback_stride + k], 2.f), 1.f);
            b.colors[3 * i + k] = (uint8_t)fminf(fmaxf(add(mul(c, 127.5f), 128.f), 0.f), 255.f);
        }
    }
}

int check_cameras(const float* cam2world, const float* intr, int views, int height, int width, const char* who) {
    N3D_CHECK_ARG(cam2world && intr, "%s: null camera buffer", who);
    N3D_CHECK_ARG(views >= 1 && height >= 1 && width >= 1, "%s: need views, height, width >= 1, got %d, %d, %d", who, views, height, width);
    N3D_CHECK_ARG(height <= (1 << 24) && width <= (1 << 24) && (int64_t)views * height * width <= (1LL << 40),
                  "%s: %d views of %dx%d pixels are too many", who, views, height, width);
    return N3D_OK;
}

}  // namespace

extern "C" int n3d_bake_world_points(const float* verts, int64_t nv, int grid_n, float cube, float* world, void* stream) {
    N3D_CHECK_ARG(nv >= 0, "n3d_bake_world_points: negative vertex count %lld", (long long)nv);
    N3D_CHECK_ARG(nv == 0 || (verts && world), "n3d_bake_world_points: null buffer");
    N3D_CHECK_ARG(grid_n >= 2, "n3d_bake_world_points: grid_n must be at least 2, got %d", grid_n);
    N3D_CHECK_ARG(isfinite(cube) && cube > 0.f, "n3d_bake_world_points: cube must be finite and positive");
    if (nv == 0) return N3D_OK;
    world_kernel<<<n3d_grid(nv, kThreads), kThreads, 0, (cudaStream_t)stream>>>(verts, nv, grid_n, cube, world);
    N3D_CHECK_LAUNCH("n3d_bake_world_points");
    return N3D_OK;
}

extern "C" int n3d_mesh_zbuffer(const float* verts, int64_t nv, const int32_t* faces, int64_t nf, const float* cam2world,
                                const float* intrinsics, int views, int height, int width, float near, uint64_t* zbuf, void* stream) {
    const char* who = "n3d_mesh_zbuffer";
    const int rc = check_cameras(cam2world, intrinsics, views, height, width, who);
    if (rc != N3D_OK) return rc;
    N3D_CHECK_ARG(zbuf, "%s: null z-buffer", who);
    N3D_CHECK_ARG((uintptr_t)zbuf % 8 == 0, "%s: the z-buffer must be 8-byte aligned", who);
    N3D_CHECK_ARG(nv >= 0 && nv < (1LL << 31) && nf >= 0 && nf < (1LL << 31), "%s: %lld vertices and %lld triangles: int32 indices "
                  "and triangle ids stop at 2^31 - 1", who, (long long)nv, (long long)nf);
    N3D_CHECK_ARG(nf == 0 || (verts && faces), "%s: null mesh buffer", who);
    N3D_CHECK_ARG(isfinite(near) && near > 0.f, "%s: the near plane must be finite and positive", who);
    const cudaStream_t s = (cudaStream_t)stream;
    const cudaError_t e = cudaMemsetAsync(zbuf, 0xff, sizeof(uint64_t) * (size_t)views * height * width, s);     // every key empty
    if (e != cudaSuccess) {
        n3d_set_error("%s: clearing the z-buffer failed: %s", who, cudaGetErrorString(e));
        return N3D_ERR_CUDA;
    }
    if (nf > 0)
        zbuffer_kernel<<<n3d_grid(nf * views, kThreads), kThreads, 0, s>>>(verts, nv, faces, nf, cam2world, intrinsics, views, height,
                                                                            width, near, (unsigned long long*)zbuf);
    N3D_CHECK_LAUNCH(who);
    return N3D_OK;
}

extern "C" int n3d_bake_vertex_colors(const float* verts, const float* world, int64_t nv, const float* grid, int grid_n,
                                      const float* cam2world, const float* intrinsics, int views, const float* images, int height,
                                      int width, const uint64_t* zbuf, float near, float eps, const float* fallback, int fallback_stride,
                                      uint8_t* colors, uint8_t* visible, float* weights, void* stream) {
    const char* who = "n3d_bake_vertex_colors";
    const int rc = check_cameras(cam2world, intrinsics, views, height, width, who);
    if (rc != N3D_OK) return rc;
    N3D_CHECK_ARG(nv >= 0, "%s: negative vertex count %lld", who, (long long)nv);
    N3D_CHECK_ARG(grid_n >= 2, "%s: grid_n must be at least 2, got %d", who, grid_n);
    N3D_CHECK_ARG(nv == 0 || (verts && world && grid && images && zbuf && fallback && colors), "%s: null buffer", who);
    N3D_CHECK_ARG(fallback_stride >= 3, "%s: fallback_stride must be at least 3, got %d", who, fallback_stride);
    N3D_CHECK_ARG(isfinite(near) && near > 0.f && isfinite(eps) && eps >= 0.f, "%s: near must be positive and eps non-negative", who);
    if (nv == 0) return N3D_OK;
    const Bake b{verts, world, grid, nv, grid_n, cam2world, intrinsics, images, views, height, width, (const unsigned long long*)zbuf,
                 near, eps, fallback, fallback_stride, colors, visible, weights};
    bake_kernel<<<n3d_grid(nv, kThreads), kThreads, 0, (cudaStream_t)stream>>>(b);
    N3D_CHECK_LAUNCH(who);
    return N3D_OK;
}
