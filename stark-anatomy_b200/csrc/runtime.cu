// runtime.cu -- library-wide state: the last error, the launch counter, the per-stream workspaces and
// the LRU of twiddle / x^-1 tables, with the C entry points that report on or release them.
#include <cstdlib>
#include <map>
#include <mutex>

#include "runtime.cuh"

using namespace sa;

thread_local std::string g_last_error;
std::atomic<uint64_t> g_launches{0};

// ------------------------------------------------------------- workspaces --
// Grow-only scratch buffers, one per (device, stream): the four-step NTT needs an n*batch
// intermediate and allocating it per call (even stream-ordered) costs more than the kernels.
static std::mutex g_ws_mu;
static std::map<std::tuple<int, cudaStream_t, int>, std::pair<void *, size_t>> g_ws;
int get_workspace(void **out, size_t bytes, cudaStream_t st, WsTag tag) {
    int dev = 0;
    SA_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_ws_mu);
    auto &slot = g_ws[std::make_tuple(dev, st, tag)];
    if (slot.second < bytes) {
        if (slot.first) {
            SA_CUDA(cudaStreamSynchronize(st));  // earlier work on this stream may still use it
            SA_CUDA(cudaFree(slot.first));
            slot.first = nullptr;
            slot.second = 0;
        }
        SA_CUDA(cudaMalloc(&slot.first, bytes));
        slot.second = bytes;
    }
    *out = slot.first;
    return SA_OK;
}
// stream-ordered pool allocations (small flags, host-entry staging) keep their memory cached
void keep_pool_memory() {
    static std::once_flag once;
    std::call_once(once, [] {
        int dev = 0;
        cudaMemPool_t pool;
        if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
            uint64_t keep = UINT64_MAX;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
    });
}

struct CacheEntry {
    std::shared_ptr<DeviceTables> tables;
    uint64_t tick = 0;
};
static std::mutex g_plan_mu;
static std::map<CacheKey, CacheEntry> g_cache;
static size_t g_cache_bytes = 0;
static size_t g_cache_limit = (size_t)4 << 30;  // bytes; SA_CACHE_LIMIT_MIB / sa_cache_limit()
static uint64_t g_cache_tick = 0;

static void cache_config() {
    static std::once_flag once;
    std::call_once(once, [] {
        if (const char *e = getenv("SA_CACHE_LIMIT_MIB")) {
            const long long v = atoll(e);
            if (v >= 0) g_cache_limit = (size_t)v << 20;
        }
    });
}
// g_plan_mu held.  Drops least-recently-used entries until `incoming` more bytes fit (an entry larger
// than the whole limit is still admitted alone: the call that needs it has to run).
static void cache_make_room(size_t incoming) {
    while (!g_cache.empty() && g_cache_bytes + incoming > g_cache_limit) {
        auto victim = g_cache.begin();
        for (auto it = g_cache.begin(); it != g_cache.end(); ++it)
            if (it->second.tick < victim->second.tick) victim = it;
        g_cache_bytes -= victim->second.tables->bytes;
        g_cache.erase(victim);  // frees the device memory once nobody holds the tables any more
    }
}
std::shared_ptr<DeviceTables> cache_find_tables(const CacheKey &key) {
    cache_config();
    std::lock_guard<std::mutex> lock(g_plan_mu);
    auto it = g_cache.find(key);
    if (it == g_cache.end()) return nullptr;
    it->second.tick = ++g_cache_tick;
    return it->second.tables;
}
// publishes `made` unless another thread got there first (then that one wins and `made` is dropped)
std::shared_ptr<DeviceTables> cache_publish_tables(const CacheKey &key, std::shared_ptr<DeviceTables> made) {
    std::lock_guard<std::mutex> lock(g_plan_mu);
    auto it = g_cache.find(key);
    if (it != g_cache.end()) {
        it->second.tick = ++g_cache_tick;
        return it->second.tables;
    }
    cache_make_room(made->bytes);
    CacheEntry e;
    e.tables = made;
    e.tick = ++g_cache_tick;
    g_cache.emplace(key, e);
    g_cache_bytes += made->bytes;
    return made;
}

extern "C" {

const char *sa_version(void) { return "sa_b200 0.1 sm_90a"; }
const char *sa_last_error(void) { return g_last_error.c_str(); }
uint64_t sa_launch_count(void) { return g_launches.load(); }

size_t sa_cache_limit(size_t bytes) {
    cache_config();
    std::lock_guard<std::mutex> lock(g_plan_mu);
    g_cache_limit = bytes;
    cache_make_room(0);
    return g_cache_bytes;
}
size_t sa_cache_bytes(void) {
    std::lock_guard<std::mutex> lock(g_plan_mu);
    return g_cache_bytes;
}
int sa_release_workspaces(void) {
    SA_CUDA(cudaDeviceSynchronize());
    int dev = 0;
    SA_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_ws_mu);
    for (auto it = g_ws.begin(); it != g_ws.end();) {
        if (std::get<0>(it->first) == dev) {
            if (it->second.first) cudaFree(it->second.first);
            it = g_ws.erase(it);
        } else {
            ++it;
        }
    }
    cudaGetLastError();
    return SA_OK;
}

}  // extern "C"
