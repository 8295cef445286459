// peer.cu -- multi-GPU assembly: CUDA IPC buffers, peer access, transforms that also store into peers'
// buffers (sa_ntt_multi) or a multicast address (sa_ntt_mcast), and the push kernels.
#include <cstdlib>
#include <cstring>

#include "ntt_tile.cuh"
#include "runtime.cuh"

using namespace sa;

// ---- multi-GPU assembly by push: one read of a finished block, one fully coalesced 16-byte store per lane
// and destination (a warp writes 512 contiguous bytes to every peer: NVLink sees whole packets, unlike the 128-byte
// segments the transform's own last pass produces)
struct PushArgs {
    uint4 *dst[TILE_MAX_PEERS];
    int ndst;
};
__global__ void __launch_bounds__(256) k_push(const __grid_constant__ PushArgs a, const uint4 *src, size_t n16) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + 3 * stride < n16; i += 4 * stride) {  // four loads in flight per thread
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) v[u] = __ldcs(src + i + u * stride);
#pragma unroll
        for (int u = 0; u < 4; u++)
#pragma unroll
            for (int p = 0; p < TILE_MAX_PEERS; p++)
                if (p < a.ndst) a.dst[p][i + u * stride] = v[u];
    }
    for (; i < n16; i += stride) {
        const uint4 v = __ldcs(src + i);
#pragma unroll
        for (int p = 0; p < TILE_MAX_PEERS; p++)
            if (p < a.ndst) a.dst[p][i] = v;
    }
}

// variant: ONE multimem.st per 16 bytes through a multicast address (NVLS): the store leaves this GPU once and the
// NVSwitch replicates it into every rank's buffer bound to the multicast object (sa_push_mcast)
__global__ void __launch_bounds__(256) k_push_mcast(fe *mc, const fe *src, size_t n16) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + 3 * stride < n16; i += 4 * stride) {
        fe v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) v[u] = tile_ld(src + i + u * stride);
#pragma unroll
        for (int u = 0; u < 4; u++) tile_st_multicast(mc + i + u * stride, v[u]);
    }
    for (; i < n16; i += stride) tile_st_multicast(mc + i, tile_ld(src + i));
}

extern "C" {

// ---- buffers shared between the processes of one box (one process per GPU) ----
int sa_peer_alloc(void **ptr, size_t bytes, uint8_t handle_out[64]) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
    *ptr = nullptr;
    SA_CUDA(cudaMalloc(ptr, bytes ? bytes : 1));  // (IPC needs a cudaMalloc allocation of its own, not a pool block)
    SA_CUDA(cudaMemset(*ptr, 0, bytes ? bytes : 1));
    cudaIpcMemHandle_t h;
    const cudaError_t e = cudaIpcGetMemHandle(&h, *ptr);
    if (e != cudaSuccess) {
        cudaFree(*ptr);
        *ptr = nullptr;
        SA_CUDA(e);
    }
    memcpy(handle_out, &h, 64);
    return SA_OK;
}
int sa_peer_open(void **ptr, const uint8_t handle[64]) {
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    *ptr = nullptr;
    // opened with THIS device current: the mapping lands in this device's address space and peer access to
    // the owner is enabled on the way, which is what lets this device's kernels store into it
    SA_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return SA_OK;
}
int sa_peer_close(void *ptr) {
    if (ptr) SA_CUDA(cudaIpcCloseMemHandle(ptr));
    return SA_OK;
}
int sa_peer_free(void *ptr) {
    if (ptr) SA_CUDA(cudaFree(ptr));
    return SA_OK;
}
int sa_copy_async(void *dst, const void *src, size_t bytes, void *stream) {
    if (bytes) SA_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
    return SA_OK;
}

int sa_ntt_mcast(void *mc, void *local, size_t out_offset, const void *in, int log_n, const uint64_t root[2],
                 int inverse, size_t batch, void *stream) {
    if (!mc || !local) return SA_ESIZE;
    return ntt_run((fe *)local + out_offset, in, log_n, root, inverse, batch, (cudaStream_t)stream, nullptr, 0,
                   (fe *)mc + out_offset);
}

int sa_push(void *const *dsts, int ndst, const void *src, size_t bytes, void *stream) {
    if (ndst < 0 || ndst > TILE_MAX_PEERS || (bytes & 15) || (((uintptr_t)src) & 15)) return SA_ESIZE;
    if (ndst == 0 || bytes == 0) return SA_OK;
    PushArgs a;
    memset(&a, 0, sizeof(a));
    a.ndst = ndst;
    for (int i = 0; i < ndst; i++) {
        if (((uintptr_t)dsts[i]) & 15) return SA_ESIZE;
        a.dst[i] = (uint4 *)dsts[i];
    }
    static const int ctas = [] {
        const char *e = getenv("SA_PUSH_CTAS");
        return e && atoi(e) > 0 ? atoi(e) : (int)sm_count();
    }();
    const size_t n16 = bytes / 16;
    size_t grid = (n16 + 255) / 256;
    if (grid > (size_t)ctas) grid = (size_t)ctas;
    k_push<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(a, (const uint4 *)src, n16);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

int sa_push_mcast(void *mc_dst, const void *src, size_t bytes, void *stream) {
    if (!mc_dst || (bytes & 15) || (((uintptr_t)src) & 15) || (((uintptr_t)mc_dst) & 15)) return SA_ESIZE;
    if (bytes == 0) return SA_OK;
    static const int ctas = [] {
        const char *e = getenv("SA_PUSH_CTAS");
        return e && atoi(e) > 0 ? atoi(e) : (int)sm_count();
    }();
    const size_t n16 = bytes / 16;
    size_t grid = (n16 + 255) / 256;
    if (grid > (size_t)ctas) grid = (size_t)ctas;
    k_push_mcast<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>((fe *)mc_dst, (const fe *)src, n16);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

int sa_enable_peer_access(int peer_device) {
    int dev = 0;
    SA_CUDA(cudaGetDevice(&dev));
    if (peer_device == dev) return SA_OK;
    int can = 0;
    SA_CUDA(cudaDeviceCanAccessPeer(&can, dev, peer_device));
    if (!can) {
        g_last_error = "sa_enable_peer_access: no peer access between these devices";
        return SA_ECUDA;
    }
    const cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) {
        cudaGetLastError();
        return SA_OK;
    }
    SA_CUDA(e);
    return SA_OK;
}

int sa_ntt_multi(void *const *outs, int nouts, size_t out_offset, const void *in, int log_n,
                 const uint64_t root[2], int inverse, size_t batch, void *stream) {
    if (nouts < 1 || nouts > TILE_MAX_PEERS + 1) return SA_ESIZE;
    fe *peers[TILE_MAX_PEERS];
    for (int i = 1; i < nouts; i++) peers[i - 1] = (fe *)outs[i] + out_offset;
    return ntt_run((fe *)outs[0] + out_offset, in, log_n, root, inverse, batch, (cudaStream_t)stream, peers,
                   nouts - 1);
}

}  // extern "C"
