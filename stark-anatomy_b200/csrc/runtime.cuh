// runtime.cuh -- internal declarations shared by the library's sources (not part of the C ABI in
// include/sa_b200.h): error reporting, the launch counter, launch helpers, workspaces and the table cache.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/sa_b200.h"
#include "field.cuh"
#include "host.cuh"

// ------------------------------------------------------------------ plumbing --
extern thread_local std::string g_last_error;
extern std::atomic<uint64_t> g_launches;

#define SA_CUDA(expr)                                                                          \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            g_last_error = std::string(#expr) + ": " + cudaGetErrorString(_e);                 \
            return SA_ECUDA;                                                                   \
        }                                                                                      \
    } while (0)
#define SA_LAUNCH_CHECK()                                                                      \
    do {                                                                                       \
        g_launches.fetch_add(1, std::memory_order_relaxed);                                    \
        cudaError_t _e = cudaGetLastError();                                                   \
        if (_e != cudaSuccess) {                                                               \
            g_last_error = std::string("kernel launch: ") + cudaGetErrorString(_e);            \
            return SA_ECUDA;                                                                   \
        }                                                                                      \
    } while (0)

// kernels with more than 48 KB of dynamic shared memory need the opt-in once per (kernel, device)
constexpr int SA_MAX_DEVICES = 64;
template <class K>
static int optin_smem(K kernel, std::atomic<bool> *done, size_t smem) {
    int dev = 0;
    SA_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= SA_MAX_DEVICES || !done[dev].load(std::memory_order_acquire)) {
        SA_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if (dev >= 0 && dev < SA_MAX_DEVICES) done[dev].store(true, std::memory_order_release);
    }
    return SA_OK;
}

// SMs of the current device, cached per device: the grid caps of the grid-stride kernels scale with it
inline long long sm_count() {
    static std::atomic<int> cached[SA_MAX_DEVICES];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= SA_MAX_DEVICES) {
        cudaGetLastError();
        dev = 0;
    }
    int n = cached[dev].load(std::memory_order_relaxed);
    if (n <= 0) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
            cudaGetLastError();
            return 132;  // (the launch that follows reports the device error)
        }
        cached[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}

static inline unsigned grid_for(long long n, int bs, int per_sm = 16) {
    long long g = (n + bs - 1) / bs;
    const long long cap = per_sm * sm_count();
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (unsigned)g;
}

// ------------------------------------------------------------- workspaces --
// grow-only scratch buffer `tag` of (current device, st).  Growing a buffer frees the old one, so a call never
// takes a tag that it or its caller still holds; distinct tags nest: sa_interpolate holds WS_INTERP_PLAN across
// the plan build (WS_PLAN_FLAG, WS_TREE) and the apply (WS_INTERP_APPLY), and every sa_ntt inside them takes WS_NTT.
enum WsTag {
    WS_NTT = 0,           // the NTT's inter-pass intermediate
    WS_HOST_STAGING = 1,  // sa_ntt_host's device copies of host buffers
    WS_PLAN_FLAG = 7,     // sa_interp_plan's zero flag
    WS_TREE = 8,          // the subproduct tree of one call (poly_tree.cuh: tree_layout)
    WS_INTERP_PLAN = 9,   // sa_interpolate's plan
    WS_INTERP_APPLY = 10  // an apply's scratch
};
int get_workspace(void **out, size_t bytes, cudaStream_t st, WsTag tag);
void keep_pool_memory();

// ---------------------------------------------------------------- table cache --
// Twiddle tables are cached per (device, log n, root, direction); FRI x^-1 tables per (device, omega, n).
// Both live in one LRU bounded by bytes (sa_cache_limit): fast_multiply's order shrinking
// (ntt.py:47-49) and a prover that walks through many domains generate new roots all the time, and
// a 2^20 plan holds a 16 MiB inter-pass matrix.  Entries are handed out as shared_ptr: an evicted
// table is freed when its last user lets go, and cudaFree waits for kernels still reading it.
struct DeviceTables {
    std::vector<void *> ptrs;
    size_t bytes = 0;
    int device = 0;
    int alloc(void **out, size_t nbytes) {
        SA_CUDA(cudaMalloc(out, nbytes));
        ptrs.push_back(*out);
        bytes += nbytes;
        return SA_OK;
    }
    ~DeviceTables() {
        if (ptrs.empty()) return;
        int cur = 0;
        const bool sw = cudaGetDevice(&cur) == cudaSuccess && cur != device && cudaSetDevice(device) == cudaSuccess;
        for (void *p : ptrs) cudaFree(p);
        if (sw) cudaSetDevice(cur);
        cudaGetLastError();
    }
};
// kind (0 plan, 1 xinv), device, log_n | n, root lo, root hi, inverse
using CacheKey = std::tuple<int, int, uint64_t, uint64_t, uint64_t, int>;
std::shared_ptr<DeviceTables> cache_find_tables(const CacheKey &key);
std::shared_ptr<DeviceTables> cache_publish_tables(const CacheKey &key, std::shared_ptr<DeviceTables> made);
template <class T>
std::shared_ptr<T> cache_find(const CacheKey &key) {
    return std::static_pointer_cast<T>(cache_find_tables(key));
}
template <class T>
std::shared_ptr<T> cache_publish(const CacheKey &key, std::shared_ptr<T> made) {
    return std::static_pointer_cast<T>(cache_publish_tables(key, made));
}

// ------------------------------------------------------------------- NTT (ntt.cu) --
// count powers base^e * lead (Montgomery form) into a new table of `owner`; swz != 0 stores them in tile_tw_slot order
int build_pow_table(DeviceTables &owner, sa::fe **out, const sa::fe &base_m, const sa::fe &lead_m, long long count,
                    cudaStream_t st, int swz = 0);
// the transform proper; `peers` (npeer <= TILE_MAX_PEERS) are extra destinations of the LAST pass: the
// same element offsets as `out`, in other GPUs' memory (sa_ntt_multi); `mc` a multicast address (sa_ntt_mcast)
int ntt_run(void *out, const void *in, int log_n, const uint64_t root[2], int inverse, size_t batch,
            cudaStream_t st, sa::fe *const *peers, int npeer, sa::fe *mc = nullptr);

// --------------------------------------------------------------- Merkle (merkle_fri.cu) --
double microbench_b2_ms(int ilp, int iters, int blocks, uint64_t *sink);
