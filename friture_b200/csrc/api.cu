// Handle lifecycle, error reporting and the NVLink peer buffers of libfrt_b200.so.
#include <cstdarg>
#include <mutex>

#include "frt_internal.cuh"

static std::string g_create_error;
static std::mutex g_create_mutex;

int frt_fail(frt_ctx *h, int code, const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (h) {
        h->err = buf;
    } else {
        std::lock_guard<std::mutex> lock(g_create_mutex);
        g_create_error = buf;
    }
    return code;
}

extern "C" int frt_version(void) { return 100; }

extern "C" int frt_create(int device, frt_handle *out) {
    if (!out) return frt_fail(nullptr, FRT_EINVAL, "frt_create: out is NULL");
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0)
        return frt_fail(nullptr, FRT_ECUDA,
                        "frt_create: no usable CUDA device (%s); friture_b200 has no CPU fallback",
                        e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    if (device < 0 || device >= count)
        return frt_fail(nullptr, FRT_EINVAL, "frt_create: device %d out of range [0,%d)", device,
                        count);
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess)
        return frt_fail(nullptr, FRT_ECUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0)
        return frt_fail(nullptr, FRT_ECUDA,
                        "frt_create: device %d is sm_%d%d; this library is built for sm_90a only",
                        device, prop.major, prop.minor);
    frt_ctx *h = new (std::nothrow) frt_ctx();
    if (!h) return frt_fail(nullptr, FRT_ENOMEM, "frt_create: out of host memory");
    h->device = device;
    h->sm_count = prop.multiProcessorCount;
    h->smem_optin = prop.sharedMemPerBlockOptin;
    *out = h;
    return FRT_OK;
}

// the handle's members free its plans, buffers, streams and events on the handle's device
extern "C" int frt_destroy(frt_handle h) {
    if (!h) return FRT_OK;
    DeviceGuard g(h->device);
    cudaDeviceSynchronize();
    delete h;
    return FRT_OK;
}

extern "C" const char *frt_last_error(frt_handle h) {
    if (h) return h->err.c_str();
    std::lock_guard<std::mutex> lock(g_create_mutex);
    return g_create_error.c_str();
}

extern "C" int frt_device_sm_count(frt_handle h) { return h ? h->sm_count : 0; }

extern "C" int64_t frt_launch_count(frt_handle h) { return h ? h->launches : 0; }

extern "C" int frt_host_alloc(frt_handle h, size_t bytes, void **out) {
    if (!h || !out) return frt_fail(h, FRT_EINVAL, "frt_host_alloc: NULL argument");
    DeviceGuard g(h->device);
    *out = nullptr;
    FRT_CUDA(h, frt_alloc_status(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocPortable), bytes));
    return FRT_OK;
}

extern "C" int frt_host_free(frt_handle h, void *p) {
    if (!p) return FRT_OK;
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CUDA(h, cudaFreeHost(p));
    return FRT_OK;
}

// ---------------------------------------------------------------- NVLink peer memory
// Buffers that other processes of the box can open (CUDA IPC) and write with the copy engines:
// the transport of the final all-gather of spectrogram columns (friture_b200/peer.py).  A plain
// cudaMalloc allocation is exportable as a whole; cudaMemcpyAsync between two devices' unified
// addresses goes over NVLink/NVSwitch without occupying an SM.
extern "C" int frt_peer_alloc(frt_handle h, size_t bytes, void **out) {
    if (!h || !out) return frt_fail(h, FRT_EINVAL, "frt_peer_alloc: NULL argument");
    DeviceGuard g(h->device);
    *out = nullptr;
    FRT_CUDA(h, frt_malloc(out, bytes ? bytes : 1));
    return FRT_OK;
}

extern "C" int frt_peer_free(frt_handle h, void *p) {
    if (!p) return FRT_OK;
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CUDA(h, cudaFree(p));
    return FRT_OK;
}

extern "C" int frt_peer_export(frt_handle h, void *p, void *handle64) {
    if (!h || !p || !handle64) return frt_fail(h, FRT_EINVAL, "frt_peer_export: NULL argument");
    DeviceGuard g(h->device);
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle is 64 bytes");
    cudaIpcMemHandle_t hd;
    FRT_CUDA(h, cudaIpcGetMemHandle(&hd, p));
    memcpy(handle64, &hd, sizeof(hd));
    return FRT_OK;
}

extern "C" int frt_peer_import(frt_handle h, const void *handle64, void **out) {
    if (!h || !handle64 || !out) return frt_fail(h, FRT_EINVAL, "frt_peer_import: NULL argument");
    DeviceGuard g(h->device);
    cudaIpcMemHandle_t hd;
    memcpy(&hd, handle64, sizeof(hd));
    *out = nullptr;
    FRT_CUDA(h, cudaIpcOpenMemHandle(out, hd, cudaIpcMemLazyEnablePeerAccess));
    return FRT_OK;
}

extern "C" int frt_peer_close(frt_handle h, void *peer_ptr) {
    if (!peer_ptr) return FRT_OK;
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CUDA(h, cudaIpcCloseMemHandle(peer_ptr));
    return FRT_OK;
}

extern "C" int frt_peer_copy(frt_handle h, void *dst, const void *src, size_t bytes, void *stream) {
    if (!h) return FRT_EINVAL;
    if (!bytes) return FRT_OK;
    if (!dst || !src) return frt_fail(h, FRT_EINVAL, "frt_peer_copy: NULL buffer");
    DeviceGuard g(h->device);
    FRT_CUDA(h, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
    return FRT_OK;
}

// One-hop all-gather push over NVLink: every CTA streams slices of this rank's block from local
// HBM (read ONCE) into the same offset of up to 15 peers' buffers with 128-bit stores.  A handful
// of CTAs keeps enough stores in flight to fill the links; each of their warps issues one load and
// n_peers stores per 512 bytes, so the kernel takes almost no issue slots from the filterbank
// kernel it overlaps (NCCL's all-gather moves the same bytes through ring steps with copy kernels
// that occupy whole SMs; the copy engines alone top out near 430 GB/s per GPU, measured).
struct PeerPushArgs {
    const float4 *src;
    float4 *dst[15];
    int n_peers;
    long long n_vec;      // float4 elements
};

__global__ void __launch_bounds__(256) peer_push_kernel(const PeerPushArgs a) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n_vec; i += 4 * stride) {
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; u++)
            if (i + u * stride < a.n_vec) v[u] = __ldcs(a.src + i + u * stride);
        for (int p = 0; p < a.n_peers; p++) {
#pragma unroll
            for (int u = 0; u < 4; u++)
                if (i + u * stride < a.n_vec) a.dst[p][i + u * stride] = v[u];
        }
    }
}

extern "C" int frt_peer_push(frt_handle h, const void *src, void *const *peer_dst, int n_peers,
                             size_t bytes, int n_ctas, void *stream) {
    if (!h) return FRT_EINVAL;
    if (!bytes || n_peers == 0) return FRT_OK;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, src && peer_dst, "NULL buffer");
    FRT_CHECK_ARG(h, n_peers >= 1 && n_peers <= 15, "n_peers must be in [1, 15]");
    FRT_CHECK_ARG(h, bytes % 16 == 0 && ((uintptr_t)src & 15) == 0, "16-byte aligned blocks only");
    PeerPushArgs a;
    a.src = reinterpret_cast<const float4 *>(src);
    for (int p = 0; p < n_peers; p++) {
        FRT_CHECK_ARG(h, peer_dst[p] && ((uintptr_t)peer_dst[p] & 15) == 0, "peer pointer NULL or unaligned");
        a.dst[p] = reinterpret_cast<float4 *>(peer_dst[p]);
    }
    a.n_peers = n_peers;
    a.n_vec = (long long)(bytes / 16);
    if (n_ctas < 1) n_ctas = 64;
    return frt_launch(h, peer_push_kernel, n_ctas, 256, 0, (cudaStream_t)stream, a);
}
