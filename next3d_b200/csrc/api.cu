// Library-level entry points and host-side state: error reporting, version, per-device facts.
#include "common.cuh"
#include <mutex>
#include <stdarg.h>

static thread_local char g_err[512] = "";

void n3d_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char* n3d_last_error(void) { return g_err; }
extern "C" int n3d_version(void) { return 100; }

static N3DDeviceState g_dev_state[128];
static std::mutex g_smem_mutex;              // guards the smem tables: entry points may be called from several host threads

N3DDeviceState* n3d_device_state(void) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 128) {
        n3d_set_error("cannot query the current CUDA device");
        return nullptr;
    }
    N3DDeviceState* d = &g_dev_state[dev];
    if (!d->num_sms) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
            n3d_set_error("cannot query the SM count of CUDA device %d", dev);
            return nullptr;
        }
        d->num_sms = n;
    }
    return d;
}

int n3d_smem_optin(const void* kernel, int bytes, const char* who) {
    N3DDeviceState* d = n3d_device_state();
    if (!d) return N3D_ERR_CUDA;
    std::lock_guard<std::mutex> lock(g_smem_mutex);
    int i = 0;
    while (i < d->n_smem && d->smem[i].kernel != kernel) ++i;
    if (i < d->n_smem && d->smem[i].bytes >= bytes) return N3D_OK;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) {
        n3d_set_error("%s: cannot raise dynamic shared memory to %d bytes: %s", who, bytes, cudaGetErrorString(e));
        return N3D_ERR_CUDA;
    }
    if (i < N3DDeviceState::kSmemSlots) {            // a full table only costs repeated calls
        d->smem[i] = {kernel, bytes};
        if (i == d->n_smem) ++d->n_smem;
    }
    return N3D_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn lookup_encode_tiled() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess) return nullptr;
    return (EncodeTiledFn)p;
}

int n3d_encode_tmap(CUtensorMap* tm, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                    const uint32_t* box, CUtensorMapSwizzle swizzle, const char* who) {
    static const EncodeTiledFn enc = lookup_encode_tiled();     // looked up once; initialisation of a static is thread-safe
    if (!enc) {
        n3d_set_error("%s: cuTensorMapEncodeTiled unavailable (no CUDA driver?)", who);
        return N3D_ERR_CUDA;
    }
    cuuint64_t gdim[5], gstr[4];
    cuuint32_t bdim[5], estr[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i]; bdim[i] = box[i]; estr[i] = 1;
        if (i < rank - 1) gstr[i] = strides[i];
    }
    const CUresult r = enc(tm, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bdim, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        n3d_set_error("%s: cuTensorMapEncodeTiled failed with CUresult %d", who, (int)r);
        return N3D_ERR_CUDA;
    }
    return N3D_OK;
}

int n3d_max_clusters(const void* kernel, int threads, int smem_bytes, int cluster, const char* who) {
    N3DDeviceState* d = n3d_device_state();
    if (!d) return 0;
    std::lock_guard<std::mutex> lock(g_smem_mutex);
    int i = 0;
    while (i < d->n_clusters && d->clusters[i].kernel != kernel) ++i;
    if (i < d->n_clusters) return d->clusters[i].clusters;
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = cluster; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.gridDim = dim3(cluster);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.attrs = &attr; cfg.numAttrs = 1;
    int n = 0;
    const cudaError_t e = cudaOccupancyMaxActiveClusters(&n, kernel, &cfg);
    if (e != cudaSuccess || n <= 0) {
        n3d_set_error("%s: cannot place clusters of %d CTAs: %s", who, cluster, e != cudaSuccess ? cudaGetErrorString(e) : "none fit");
        return 0;
    }
    if (i < N3DDeviceState::kSmemSlots) {
        d->clusters[i] = {kernel, n};
        ++d->n_clusters;
    }
    return n;
}
