// ntt.cu -- the NTT: the tile kernel, the twiddle-table kernels, plans, tile launch, and the device
// (sa_ntt) and host-buffer (sa_ntt_host, sa_host_alloc) entry points.
//
// Reference behaviour reproduced (bit-exact): code/ntt.py:3-30.
#include <pthread.h>
#include <sched.h>

#include <algorithm>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "ntt_plan.cuh"
#include "ntt_tile.cuh"
#include "runtime.cuh"

using namespace sa;

// ------------------------------------------------------------------- kernels --
template <int LOGL, int ELOG, int C>
struct TileLaunch {
    using P = TilePlan<LOGL, ELOG, C>;
    // aim for 1024 resident threads per SM with 8-element blocks (<= 64 registers) and 512 with
    // 16-element blocks (<= 128 registers)
    static constexpr int TARGET = (P::EL <= 3 && LOGL > 3) ? 1024 : 512;
    static constexpr int MINB = TARGET / P::THREADS > 0 ? TARGET / P::THREADS : 1;
};

template <int LOGL, int ELOG, int C, int FLAGS>
__global__ void __launch_bounds__(TilePlan<LOGL, ELOG, C>::THREADS, TileLaunch<LOGL, ELOG, C>::MINB)
    ntt_tile_kernel(const __grid_constant__ TileArgs a, long long total_tiles, int tiles_per_batch) {
    using P = TilePlan<LOGL, ELOG, C>;
    using S = TileStages<LOGL, ELOG, C, FLAGS>;
    extern __shared__ uint4 sa_smem_u4[];
    fe *smem = reinterpret_cast<fe *>(sa_smem_u4);
    const int tic = threadIdx.x / P::TPT, t = threadIdx.x % P::TPT;
    const long long tile = (long long)blockIdx.x * P::TPC + tic;
    const bool valid = tile < total_tiles;
    const long long b = valid ? tile / tiles_per_batch : 0;
    const int col0 = valid ? (int)(tile % tiles_per_batch) * C : 0;
    fe *sm = smem + (size_t)tic * P::L * C;
    fe *tw = nullptr;
    uint64_t *bar = nullptr;
    // programmatic dependent launch: the next launch on this stream (pass 2 after pass 1, the next transform
    // of a chain) may become resident while this grid still runs; it parks at griddepcontrol.wait below
    asm volatile("griddepcontrol.launch_dependents;");
    if constexpr (P::NLOOP > 0) {
        // stage the twiddle table of this tile length into shared memory (bulk-async copy + mbarrier);
        // the table is a cached constant of the plan, not an output of the preceding launch
        tw = smem + P::TILE_BYTES / sizeof(fe);
        bar = reinterpret_cast<uint64_t *>(tw + P::L);
        if (threadIdx.x == 0) tile_stage_twiddles(tw, a.tw, (uint32_t)P::TW_BYTES, bar);
        __syncthreads();  // the barrier is initialised before anybody polls it
    }
    // everything the preceding launch wrote (the intermediate of the four-step split, or this call's input)
    // is complete and visible after this point; a no-op for a launch without the PDL attribute
    asm volatile("griddepcontrol.wait;" ::: "memory");
#pragma unroll 1
    for (int st = 0; st < P::NLOOP; st++) {
        S::full(st, t, sm, a, b, col0, valid, tw, bar);
        __syncthreads();
    }
    S::last(t, sm, a, b, col0, valid);
}

// one thread per 16 entries of a power table / an inter-pass matrix (ntt_plan.cuh)
__global__ void k_pow_table(fe *out, fe base_m, fe lead_m, long long count, int swz) {
    ntt_pow_table_thread(out, base_m, lead_m, count, swz, (long long)blockIdx.x * blockDim.x + threadIdx.x);
}
__global__ void k_twb_table(fe *out, fe w_m, fe scale_m, int n1, int n2) {
    ntt_twb_table_thread(out, w_m, scale_m, n1, n2, (long long)blockIdx.x * blockDim.x + threadIdx.x);
}

// ---------------------------------------------------------------- NTT plans --
struct NttPlan : DeviceTables, NttTables {
    NttShape shape;
};
using PlanPtr = std::shared_ptr<NttPlan>;

int build_pow_table(DeviceTables &owner, fe **out, const fe &base_m, const fe &lead_m, long long count,
                    cudaStream_t st, int swz) {
    int rc = owner.alloc((void **)out, sizeof(fe) * (size_t)count);
    if (rc != SA_OK) return rc;
    const long long threads = (count + 15) / 16;
    const int bs = 128;
    k_pow_table<<<(unsigned)((threads + bs - 1) / bs), bs, 0, st>>>(*out, base_m, lead_m, count, swz);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

// validates the root like ntt.py:10-11 and returns (creating if needed) the plan.  Tables are built
// outside the cache lock; a failed build frees what it had allocated (the plan object owns them).
static int get_plan(PlanPtr *plan_out, int log_n, const fe &root, int inverse, cudaStream_t st) {
    int dev = 0;
    SA_CUDA(cudaGetDevice(&dev));
    const uint64_t rlo = (uint64_t)root.v[0] | ((uint64_t)root.v[1] << 32);
    const uint64_t rhi = (uint64_t)root.v[2] | ((uint64_t)root.v[3] << 32);
    const CacheKey key(0, dev, (uint64_t)log_n, rlo, rhi, inverse ? 1 : 0);
    if ((*plan_out = cache_find<NttPlan>(key))) return SA_OK;
    const fe root_m = fe_to_mont(root);
    int rc = ntt_check_root(root_m, log_n);
    if (rc != SA_OK) return rc;
    PlanPtr made = std::make_shared<NttPlan>();
    NttPlan &p = *made;
    p.device = dev;
    p.shape = ntt_shape(log_n);
    auto pow = [&](fe **out, const fe &base_m, long long count) -> int {
        return build_pow_table(p, out, base_m, fe_mont_one(), count, st, 1);
    };
    auto twb = [&](fe **out, const fe &w_m, const fe &scale_m, int rows, long long cols) -> int {
        const int rc = p.alloc((void **)out, sizeof(fe) * (size_t)rows * (size_t)cols);
        if (rc != SA_OK) return rc;
        const long long threads = (long long)rows * ((cols + 15) / 16);
        const int bs = 128;
        k_twb_table<<<(unsigned)((threads + bs - 1) / bs), bs, 0, st>>>(*out, w_m, scale_m, rows, (int)cols);
        SA_LAUNCH_CHECK();
        return SA_OK;
    };
    if ((rc = ntt_build_tables(p, p.shape, root_m, inverse, pow, twb)) != SA_OK) return rc;
    // the tables were built on `st`; other streams may pick the plan up from the cache right away,
    // so they must be complete before it is published (one-time cost per plan)
    SA_CUDA(cudaStreamSynchronize(st));
    *plan_out = cache_publish<NttPlan>(key, made);
    return SA_OK;
}

template <int LOGL, int ELOG, int C, int FLAGS>
static int launch_tile_variant(const TileArgs &a, cudaStream_t st) {
    using P = TilePlan<LOGL, ELOG, C>;
    const int tiles_per_batch = (a.ncols + C - 1) / C;
    const long long total = (long long)tiles_per_batch * a.nbatch;
    const long long grid = (total + P::TPC - 1) / P::TPC;
    const size_t smem = P::smem_bytes();
    if (smem > 48 * 1024) {
        static std::atomic<bool> attr_done[SA_MAX_DEVICES];
        const int rc = optin_smem(ntt_tile_kernel<LOGL, ELOG, C, FLAGS>, attr_done, smem);
        if (rc != SA_OK) return rc;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(P::THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const int tpb = tiles_per_batch;
    SA_CUDA(cudaLaunchKernelEx(&cfg, ntt_tile_kernel<LOGL, ELOG, C, FLAGS>, a, total, tpb));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return SA_OK;
}
template <int LOGL, int ELOG, int C>
static int launch_tile(const TileArgs &a, cudaStream_t st) {
    const int variant = tile_variant<LOGL, ELOG, C>(a);
    if (variant & TF_TWB2) {
        // factored pass-1 twiddles exist only above 2^26, where pass 1 runs 2^9- or 2^10-point tiles in the
        // shape launch_tile_shape gives a pass without peers (tuning shapes of -DSA_TUNE do not have them)
        if constexpr (LOGL >= 9 && ELOG == 4 && C == 4) {
            if (variant & TF_FULL) return launch_tile_variant<LOGL, ELOG, C, TF_FULL | TF_TWB2>(a, st);
            return launch_tile_variant<LOGL, ELOG, C, TF_DYNAMIC | TF_TWB2>(a, st);
        }
        return SA_ESIZE;
    }
    if constexpr (LOGL >= 5) {
        switch (variant) {
            case TF_FULL | TF_TWB: return launch_tile_variant<LOGL, ELOG, C, TF_FULL | TF_TWB>(a, st);
            case TF_FULL: return launch_tile_variant<LOGL, ELOG, C, TF_FULL>(a, st);
            case TF_FULL | TF_PEERS: return launch_tile_variant<LOGL, ELOG, C, TF_FULL | TF_PEERS>(a, st);
        }
    }
    if (variant & TF_PEERS) return launch_tile_variant<LOGL, ELOG, C, TF_DYNAMIC | TF_PEERS>(a, st);
    return launch_tile_variant<LOGL, ELOG, C, TF_DYNAMIC>(a, st);
}

// tile shape: register block (log2 elements per thread) and columns per tile; with -DSA_TUNE
// the environment variables SA_NTT_ELOG / SA_NTT_C select a shape for tuning runs.
static int g_tile_elog = -1, g_tile_c = -1;
static void tile_config() {
    if (g_tile_elog >= 0) return;
    const char *e = getenv("SA_NTT_ELOG"), *c = getenv("SA_NTT_C");
    g_tile_elog = e ? atoi(e) : 0;
    g_tile_c = c ? atoi(c) : 0;
}
template <int LOGL>
static int launch_tile_shape(const TileArgs &a, cudaStream_t st) {
    tile_config();
#ifdef SA_TUNE
    if (LOGL >= 9 && g_tile_elog > 0) {
        if (g_tile_elog == 3 && g_tile_c == 8) return launch_tile<LOGL, 3, 8>(a, st);
        if (g_tile_elog == 3 && g_tile_c == 4) return launch_tile<LOGL, 3, 4>(a, st);
        if (g_tile_elog == 3 && g_tile_c == 2) return launch_tile<LOGL, 3, 2>(a, st);
        if (g_tile_elog == 4 && g_tile_c == 4) return launch_tile<LOGL, 4, 4>(a, st);
        if (g_tile_elog == 4 && g_tile_c == 2) return launch_tile<LOGL, 4, 2>(a, st);
        if (g_tile_elog == 4 && g_tile_c == 8) return launch_tile<LOGL, 4, 8>(a, st);
    }
#endif
    // with the stage twiddles in shared memory, 16-element register blocks on 4-column tiles (2 CTAs x 256
    // threads per SM, <= 128 registers each) for the big tiles; the other shapes stay selectable for tuning
    // runs (-DSA_TUNE above)
    if constexpr (LOGL >= 9) {
        // multi-GPU assembly (sa_ntt_multi): 8-column tiles store 128-byte instead of 64-byte segments to the
        // peers, and that pass is bound by the links, not by the butterflies
        if (a.npeer > 0 || a.mc_out != nullptr) return launch_tile<LOGL, 4, 8>(a, st);
        // (a LONE 2^20 transform is one partial wave per pass: 256 four-column tiles on two CTA slots per SM.
        // Evening the columns out - seven-column tiles, one 14-warp CTA per SM, or a mixed grid of four- and
        // three-column tiles - was tried and lost: a lone pass is bound by the latency of a tile's own dependent
        // phases, not by the busiest SM's column count.)
        return launch_tile<LOGL, 4, 4>(a, st);
    }
    return launch_tile<LOGL, 4, 8>(a, st);
}
static int launch_tile_dyn(int logl, const TileArgs &a, cudaStream_t st) {
    switch (logl) {
        case 1: return launch_tile_shape<1>(a, st);
        case 2: return launch_tile_shape<2>(a, st);
        case 3: return launch_tile_shape<3>(a, st);
        case 4: return launch_tile_shape<4>(a, st);
        case 5: return launch_tile_shape<5>(a, st);
        case 6: return launch_tile_shape<6>(a, st);
        case 7: return launch_tile_shape<7>(a, st);
        case 8: return launch_tile_shape<8>(a, st);
        case 9: return launch_tile_shape<9>(a, st);
        case 10: return launch_tile_shape<10>(a, st);
    }
    return SA_ESIZE;
}

int ntt_run(void *out, const void *in, int log_n, const uint64_t root[2], int inverse, size_t batch,
            cudaStream_t st, fe *const *peers, int npeer, fe *mc) {
    if (log_n < 0 || log_n > NTT_MAX_LOG_N) return SA_ESIZE;
    if (batch == 0) return SA_OK;
    const size_t n = size_t(1) << log_n;
    if (log_n == 0) {  // ntt.py:5-6 / :23-24: a length-1 sequence is returned as is
        if (out != in) SA_CUDA(cudaMemcpyAsync(out, in, 16 * batch, cudaMemcpyDeviceToDevice, st));
        for (int i = 0; i < npeer; i++)
            SA_CUDA(cudaMemcpyAsync(peers[i], in, 16 * batch, cudaMemcpyDeviceToDevice, st));
        if (mc) return SA_ESIZE;  // (no kernel runs for length-1 transforms: not offered through a multicast address)
        return SA_OK;
    }
    PlanPtr p;  // keeps the tables alive until the launches below are enqueued (cudaFree waits for them)
    int rc = get_plan(&p, log_n, fe_from_limbs(root), inverse, st);
    if (rc != SA_OK) return rc;
    const NttShape &shape = p->shape;
    fe *tmp = nullptr;
    if (shape.l2 == 0) {
        // every transform is one tile column; in-place is safe because a tile reads all of
        // its columns into registers before it writes any of them
        if (batch > (size_t)1 << 30) return SA_ESIZE;
    } else {
        if ((rc = get_workspace((void **)&tmp, sizeof(fe) * n * batch, st, WS_NTT)) != SA_OK) return rc;
        if (shape.l3 > 0 && batch * ((size_t)1 << (shape.l1 > shape.l2 ? shape.l1 : shape.l2)) > ((size_t)1 << 30))
            return SA_ESIZE;
    }
    return ntt_run_passes(shape, *p, (const fe *)in, (fe *)out, tmp, batch, [&](int logl, TileArgs &a, bool last) {
        if (last) {
            a.npeer = npeer;
            for (int i = 0; i < npeer; i++) a.peer_out[i] = peers[i];
            a.mc_out = mc;
        }
        return launch_tile_dyn(logl, a, st);
    });
}

extern "C" {

int sa_ntt(void *out, const void *in, int log_n, const uint64_t root[2], int inverse, size_t batch,
           void *stream) {
    return ntt_run(out, in, log_n, root, inverse, batch, (cudaStream_t)stream, nullptr, 0);
}

// Host entry: H2D, transforms, D2H.  Batches are cut into chunks of a few transforms that rotate over
// a few internal streams so that the upload of chunk i+1, the kernels of chunk i and the download
// of chunk i-1 overlap (PCIe is full duplex); with pinned host buffers the call is bound by the
// slower copy direction instead of the sum of both.
constexpr int HOST_STREAMS_MAX = 8;
// one set of copy streams (and of the device buffers that go with them) per device; a set is used by
// one sa_ntt_host call at a time - the link is the shared resource anyway
struct CopySet {
    cudaStream_t streams[HOST_STREAMS_MAX];
    cudaEvent_t events[HOST_STREAMS_MAX + 1];
    std::mutex busy;
};
static std::map<int, CopySet *> g_copy_sets;
static std::mutex g_copy_mu;
static int g_host_streams = 4;            // SA_HOST_STREAMS
static size_t g_host_chunk = 32u << 20;   // SA_HOST_CHUNK_MIB: bytes per pipelined chunk
static int g_host_ramp = 1;               // SA_HOST_RAMP: first/last chunks start at chunk >> ramp
// (tools/e2e_sweep.py compares settings; a few large chunks with short ramps keep both copy directions busy)
static int get_copy_set(CopySet **out) {
    int dev = 0;
    SA_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_copy_mu);
    auto it = g_copy_sets.find(dev);
    if (it != g_copy_sets.end()) {
        *out = it->second;
        return SA_OK;
    }
    static bool configured = false;
    if (!configured) {
        configured = true;
        if (const char *e = getenv("SA_HOST_STREAMS")) {
            const int v = atoi(e);
            if (v >= 1 && v <= HOST_STREAMS_MAX) g_host_streams = v;
        }
        if (const char *e = getenv("SA_HOST_CHUNK_MIB")) {
            const int v = atoi(e);
            if (v >= 1 && v <= 1024) g_host_chunk = (size_t)v << 20;
        }
        if (const char *e = getenv("SA_HOST_RAMP")) {
            const int v = atoi(e);
            if (v >= 0 && v <= 6) g_host_ramp = v;
        }
    }
    CopySet *set = new CopySet();
    for (int i = 0; i < g_host_streams; i++)
        SA_CUDA(cudaStreamCreateWithFlags(&set->streams[i], cudaStreamNonBlocking));
    for (int i = 0; i <= g_host_streams; i++)
        SA_CUDA(cudaEventCreateWithFlags(&set->events[i], cudaEventDisableTiming));
    g_copy_sets[dev] = set;
    *out = set;
    return SA_OK;
}

int sa_ntt_host(void *out_host, const void *in_host, int log_n, const uint64_t root[2], int inverse,
                size_t batch, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (log_n < 0 || log_n > NTT_MAX_LOG_N) return SA_ESIZE;
    const size_t one = size_t(16) << log_n;
    const size_t bytes = one * batch;
    if (bytes == 0) return SA_OK;
    int rc;
    if (log_n > NTT_FULL_TWB_MAX_LOG_N) {
        // a transform above 2^26 is a chunk of its own, and every pipelined chunk would hold a staging buffer
        // and an n-element intermediate per copy stream (32 GiB at 2^28): one transform at a time instead,
        // through one staging buffer on `st`
        void *dev = nullptr;
        if ((rc = get_workspace(&dev, one, st, WS_HOST_STAGING)) != SA_OK) return rc;
        for (size_t b = 0; b < batch && rc == SA_OK; b++) {
            SA_CUDA(cudaMemcpyAsync(dev, (const char *)in_host + b * one, one, cudaMemcpyHostToDevice, st));
            rc = sa_ntt(dev, dev, log_n, root, inverse, 1, stream);
            if (rc == SA_OK) SA_CUDA(cudaMemcpyAsync((char *)out_host + b * one, dev, one, cudaMemcpyDeviceToHost, st));
        }
        SA_CUDA(cudaStreamSynchronize(st));
        return rc;
    }
    CopySet *cset = nullptr;
    if ((rc = get_copy_set(&cset)) != SA_OK) return rc;
    // chunk = as many transforms as fit g_host_chunk (default two 2^20 transforms); small jobs stay on `st`
    size_t per_chunk = one >= g_host_chunk ? 1 : g_host_chunk / one;
    if (per_chunk > batch) per_chunk = batch;
    const size_t nchunks = (batch + per_chunk - 1) / per_chunk;
    if (nchunks < 2) {
        void *dev = nullptr;
        if ((rc = get_workspace(&dev, bytes, st, WS_HOST_STAGING)) != SA_OK) return rc;
        SA_CUDA(cudaMemcpyAsync(dev, in_host, bytes, cudaMemcpyHostToDevice, st));
        rc = sa_ntt(dev, dev, log_n, root, inverse, batch, stream);
        if (rc == SA_OK) SA_CUDA(cudaMemcpyAsync(out_host, dev, bytes, cudaMemcpyDeviceToHost, st));
        SA_CUDA(cudaStreamSynchronize(st));
        return rc;
    }
    const int ns = g_host_streams;
    std::lock_guard<std::mutex> one_call_at_a_time(cset->busy);
    cudaStream_t *g_copy_streams = cset->streams;
    cudaEvent_t *g_copy_events = cset->events;
    // chunk sizes (in transforms): ramp up from a small first chunk and down to a small last one, so
    // that the stretch where only one copy direction is busy (before the first kernel can start, after
    // the last one has finished) is short while the bulk moves in few large copies
    std::vector<size_t> counts;
    {
        std::vector<size_t> head;
        // (per_chunk <= 1 has nothing to ramp; the start is clamped so that c <<= 1 always makes progress)
        if (g_host_ramp && per_chunk > 1)
            for (size_t c = std::max<size_t>(1, per_chunk >> g_host_ramp); c < per_chunk; c <<= 1) head.push_back(c);
        size_t ramp = 0;
        for (size_t c : head) ramp += c;
        if (2 * ramp >= batch) head.clear(), ramp = 0;
        counts = head;
        for (size_t left = batch - 2 * ramp; left > 0;) {
            const size_t c = left < per_chunk ? left : per_chunk;
            counts.push_back(c);
            left -= c;
        }
        counts.insert(counts.end(), head.rbegin(), head.rend());
    }
    void *buf[HOST_STREAMS_MAX];
    for (int i = 0; i < ns; i++)
        if ((rc = get_workspace(&buf[i], per_chunk * one, g_copy_streams[i], WS_HOST_STAGING)) != SA_OK) return rc;
    SA_CUDA(cudaEventRecord(g_copy_events[ns], st));
    for (int i = 0; i < ns; i++) SA_CUDA(cudaStreamWaitEvent(g_copy_streams[i], g_copy_events[ns], 0));
    rc = SA_OK;
    size_t first = 0;
    for (size_t c = 0; c < counts.size() && rc == SA_OK; c++) {
        const int si = (int)(c % ns);
        cudaStream_t cs = g_copy_streams[si];
        const size_t cnt = counts[c];
        const char *src = (const char *)in_host + first * one;
        char *dst = (char *)out_host + first * one;
        first += cnt;
        // within one stream the copies and kernels of successive chunks are ordered, so one device
        // buffer per stream is enough; different streams overlap upload, kernels and download
        SA_CUDA(cudaMemcpyAsync(buf[si], src, cnt * one, cudaMemcpyHostToDevice, cs));
#ifdef SA_TUNE
        static const bool skip_ntt = getenv("SA_HOST_SKIP_NTT") != nullptr;  // copy pipeline alone (diagnostic)
        if (!skip_ntt)
#endif
        rc = sa_ntt(buf[si], buf[si], log_n, root, inverse, cnt, (void *)cs);
        if (rc == SA_OK) SA_CUDA(cudaMemcpyAsync(dst, buf[si], cnt * one, cudaMemcpyDeviceToHost, cs));
    }
    for (int i = 0; i < ns; i++) {
        SA_CUDA(cudaEventRecord(g_copy_events[i], g_copy_streams[i]));
        SA_CUDA(cudaStreamWaitEvent(st, g_copy_events[i], 0));
    }
    SA_CUDA(cudaStreamSynchronize(st));
    return rc;
}

// ---- pinned host buffers next to the GPU ----
static bool gpu_local_cpus(cpu_set_t *set) {
    int dev = 0;
    char bdf[32] = {0};
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetPCIBusId(bdf, sizeof(bdf), dev) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    for (char *c = bdf; *c; c++) *c = (char)tolower((unsigned char)*c);
    const std::string path = std::string("/sys/bus/pci/devices/") + bdf + "/local_cpulist";
    FILE *f = fopen(path.c_str(), "r");
    if (!f) return false;
    char text[4096] = {0};
    const size_t got = fread(text, 1, sizeof(text) - 1, f);
    fclose(f);
    if (got == 0) return false;
    CPU_ZERO(set);
    int count = 0;
    for (char *tok = strtok(text, ",\n"); tok; tok = strtok(nullptr, ",\n")) {  // "0-31,64-95"
        int a = 0, b = 0;
        const int k = sscanf(tok, "%d-%d", &a, &b);
        if (k < 1) continue;
        if (k == 1) b = a;
        for (int c = a; c <= b && c < CPU_SETSIZE; c++, count++) CPU_SET(c, set);
    }
    return count > 0;
}

void *sa_host_alloc(size_t bytes) {
    if (bytes == 0) bytes = 1;
    cpu_set_t before, near, both;
    const bool have_before = pthread_getaffinity_np(pthread_self(), sizeof(before), &before) == 0;
    bool moved = false;
    if (have_before && gpu_local_cpus(&near)) {
        CPU_AND(&both, &before, &near);
        if (CPU_COUNT(&both) > 0) moved = pthread_setaffinity_np(pthread_self(), sizeof(both), &both) == 0;
    }
    void *p = nullptr;
    const cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocPortable);  // pages are placed now, here
    if (e == cudaSuccess) memset(p, 0, bytes);
    if (moved) pthread_setaffinity_np(pthread_self(), sizeof(before), &before);
    if (e != cudaSuccess) {
        g_last_error = std::string("sa_host_alloc: ") + cudaGetErrorString(e);
        cudaGetLastError();
        return nullptr;
    }
    return p;
}

int sa_host_free(void *p) {
    if (p) SA_CUDA(cudaFreeHost(p));
    return SA_OK;
}

}  // extern "C"
