// merkle_fri.cu -- Merkle trees, openings, gathers and FRI: fold, fused fold + tree rounds and the
// whole commit with per-round challenges from the host.
//
// Reference behaviour reproduced (bit-exact): code/fri.py:85, code/merkle.py:6-27.
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>

#include "fri_merkle.cuh"
#include "hash.cuh"
#include "ntt_tile.cuh"
#include "runtime.cuh"

using namespace sa;

__global__ void k_fri_fold(fe *next, const fe *cw, long long half, const fe *xinv, fe s_m, fe inv2_m) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += stride) {
        const fe t_m = fe_montmul(tile_ldg(xinv + i), s_m);
        tile_st(next + i, fri_fold_one(tile_ld(cw + i), tile_ld(cw + half + i), t_m, inv2_m));
    }
}

// the host waits for the root of every FRI round before it can draw the next challenge: the last CTA
// of a tree writes it straight into mapped host memory, followed (system-scope fence) by a sequence
// number the host spins on - no copy engine, no stream synchronisation on the critical path
__device__ __forceinline__ void merkle_publish_root(const MerkleArgs &a, const uint64_t *root) {
    volatile uint64_t *out = a.root_out;
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = root[i];
    __threadfence_system();
    out[8] = a.root_seq;
}
// One CTA reduces `chunk` bottom nodes to one node, writing every level to the heap-ordered tree.
// Phase 1: every thread reduces its 2^ipt_log bottom nodes privately (no barrier); phase 2: the
// per-thread digests are reduced through shared memory.  mode 2 is the fused FRI round:
// fold -> leaf digest -> subtree, one pass over the codeword.
// The 2 in __launch_bounds__ is the minimum of resident CTAs per SM, i.e. at most 128 registers: without
// the bound the kernel drifts above 128 registers and only one CTA fits per SM.
// A batch of trees of one width is one launch: blockIdx.y is the tree, so gridDim.x stays the CTA count
// of one tree and the launch shape, the fused top's arrival count and the heap indices are those of a
// single tree.
__global__ void __launch_bounds__(MK_THREADS, 2) k_merkle_chunk(const __grid_constant__ MerkleArgs args) {
    __shared__ uint64_t sm[MK_THREADS * 8];
    const MerkleArgs a = merkle_tree_args(args, blockIdx.y);
    const long long blk = blockIdx.x;
    const unsigned nblocks = gridDim.x;
    const int tid = threadIdx.x;
    if (a.mode == 1 && blk == 0 && tid < 8) a.tree[tid] = 0;  // the unused node 0
    const int active = a.chunk >> a.ipt_log;  // threads with a private subtree
    uint64_t d[8];
    if (tid < active) merkle_private(d, a, blk, tid);
    if (a.red_log == 0) {  // the next launch picks the subtree roots up from the tree
        if (a.root_out && tid == 0) merkle_publish_root(a, d);  // (a tree of one leaf)
        return;
    }
    if (tid < active) {
#pragma unroll
        for (int i = 0; i < 8; i++) sm[tid * 8 + i] = d[i];
    }
    __syncthreads();
    // index of thread 0's subtree root; the level above it starts at base >> 1, and so on
    long long base = (a.width + blk * a.chunk) >> a.ipt_log;
    int wl = active / 2, levels = a.red_log, coop_max = a.coop_max;
    for (int pass = 0;; pass++) {
        for (int lvl = 0; lvl < levels; wl >>= 1, lvl++) {
            base >>= 1;
            if (wl > coop_max || wl > MK_THREADS / 4) {  // plenty of nodes: one thread per node
                const bool mine = tid < wl;
                if (mine) merkle_node_digest(d, sm + (2 * tid) * 8, sm + (2 * tid + 1) * 8);
                __syncthreads();
                if (mine) {
                    uint64_t *node = a.tree + (base + tid) * 8;
#pragma unroll
                    for (int i = 0; i < 8; i++) {
                        sm[tid * 8 + i] = d[i];
                        node[i] = d[i];
                    }
                }
            } else {  // few nodes, the level is a dependency chain: four lanes per node (hash.cuh)
                const int q = tid >> 2, j = tid & 3;
                const bool warp_on = (tid >> 5) < ((4 * wl + 31) >> 5);  // whole warps only (shuffles)
                uint64_t lo = 0, hi = 0;
                if (warp_on) blake2b_coop4_node(lo, hi, sm + (2 * (q < wl ? q : 0)) * 8, j);
                __syncthreads();
                if (warp_on && q < wl) {
                    uint64_t *node = a.tree + (base + q) * 8;
                    sm[q * 8 + j] = lo;
                    sm[q * 8 + 4 + j] = hi;
                    node[j] = lo;
                    node[4 + j] = hi;
                }
            }
            __syncthreads();
        }
        if (pass == 1 || a.ticket == nullptr) break;
        // Every CTA of this tree has reduced its chunk to one digest (heap node nblocks + blk).  The
        // CTA that arrives last reduces those nblocks digests as well instead of leaving them to one
        // more launch (each thread fences its own stores, the barrier orders them before the ticket).
        __shared__ int s_last;
        __threadfence();
        __syncthreads();
        if (tid == 0) s_last = atomicAdd(a.ticket, 1u) == nblocks - 1;
        __syncthreads();
        if (!s_last) return;
        const int g = (int)nblocks;
        if (tid == 0) *a.ticket = 0;  // as the next launch on this stream expects it
        __threadfence();
        if (tid < g) {
            const uint64_t *node = a.tree + (size_t)(g + tid) * 8;
#pragma unroll
            for (int i = 0; i < 8; i++) sm[tid * 8 + i] = __ldcg(node + i);  // written by other SMs: not via L1
        }
        __syncthreads();
        base = g;
        wl = g / 2;
        levels = 31 - __clz(g);
        coop_max = MK_THREADS / 4;  // this part is a dependency chain whatever the shape below was
    }
    if (a.root_out && tid == 0) merkle_publish_root(a, sm);
}

// out[b][q][level] = word w of the sibling at `level` of the leaf index q of tree b's set, in tree b
__global__ void k_merkle_paths(uint64_t *out, const uint64_t *trees, long long n, int depth,
                               const uint64_t *indices, long long k, long long batch, long long group) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < batch * k * depth * 8) merkle_path_sets_elem(out, trees, n, depth, indices, k, group, t);
}
// out[b][q] = values[b * n + the index q of row b's set]
__global__ void k_gather(fe *out, const fe *values, long long n, const uint64_t *indices, long long k,
                         long long batch, long long group) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < batch * k) gather_sets_elem(out, values, n, indices, k, group, t);
}

// blake2b-only roof of the Merkle kernels: every thread hashes a chain of node messages (128 bytes = one
// compression each, merkle.py:11) that never leave its registers
template <int ILP>
__global__ void __launch_bounds__(MK_THREADS) k_microbench_b2(uint64_t *sink, int iters) {
    uint64_t d[ILP][8];
    const uint64_t t = blockIdx.x * blockDim.x + threadIdx.x;
#pragma unroll
    for (int i = 0; i < ILP; i++)
#pragma unroll
        for (int k = 0; k < 8; k++) d[i][k] = t * 0x9E3779B97F4A7C15ull + 131 * i + k;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) merkle_node_digest(d[i], d[i], d[(i + 1) % ILP]);
    }
    uint64_t acc = 0;
#pragma unroll
    for (int i = 0; i < ILP; i++)
#pragma unroll
        for (int k = 0; k < 8; k++) acc ^= d[i][k];
    if (acc == 0x1234567ull) sink[t] = acc;
}

// sa_microbench op 4 (threads is fixed at MK_THREADS): blake2b node compressions in ms.  It sits next to
// k_merkle_chunk so that both callers of the noinline blake2b_single_block are compiled in one module, as
// in the Merkle kernels it is the roof of.
double microbench_b2_ms(int ilp, int iters, int blocks, uint64_t *sink) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    auto run = [&](int it) {
        if (ilp >= 2)
            k_microbench_b2<2><<<blocks, MK_THREADS>>>(sink, it);
        else
            k_microbench_b2<1><<<blocks, MK_THREADS>>>(sink, it);
    };
    run(iters / 8 + 1);
    cudaEventRecord(e0);
    run(iters);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float f = 0;
    cudaEventElapsedTime(&f, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return (double)f;
}

struct XinvTable : DeviceTables {
    fe *tab = nullptr;
};
using XinvPtr = std::shared_ptr<XinvTable>;

// ---- Merkle / FRI ----
// arrival counters of k_merkle_chunk's fused top, one per tree of a launch, per (device, stream): zero
// whenever no launch of that stream is in flight (the last CTA of a tree resets its counter).  They grow
// in 256-byte steps and never shrink.
struct Tickets {
    unsigned int *ptr = nullptr;
    int count = 0;
};
static std::mutex g_tickets_mu;
static std::map<std::pair<int, cudaStream_t>, Tickets> g_tickets;
static unsigned int *get_tickets(cudaStream_t st, int trees) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
    std::lock_guard<std::mutex> lock(g_tickets_mu);
    Tickets &slot = g_tickets[std::make_pair(dev, st)];
    if (slot.count < trees) {
        const int count = (trees + 63) / 64 * 64;
        // earlier launches on this stream may still count on the old counters
        if (slot.ptr && (cudaStreamSynchronize(st) != cudaSuccess || cudaFree(slot.ptr) != cudaSuccess)) {
            cudaGetLastError();
            return nullptr;  // (the counters stay as they are)
        }
        slot = Tickets();
        if (cudaMalloc((void **)&slot.ptr, 4 * (size_t)count) != cudaSuccess ||
            cudaMemsetAsync(slot.ptr, 0, 4 * (size_t)count, st) != cudaSuccess) {
            if (slot.ptr) cudaFree(slot.ptr);
            slot = Tickets();
            cudaGetLastError();
        } else {
            slot.count = count;
        }
    }
    return slot.ptr;  // nullptr: fall back to one more launch
}
// the launches of `batch` trees, merkle_view's layout; root_host: tree b publishes its root at root_host + 9 b
static int merkle_reduce(MerkleArgs a, size_t batch, cudaStream_t st, uint64_t *root_host = nullptr,
                         unsigned long long seq = 0) {
#ifdef SA_TUNE
    const char *shape_spec = getenv("SA_MK_SHAPE");  // see merkle_shape_override
#else
    const char *shape_spec = nullptr;
#endif
    a.root_out = root_host;  // (merkle_view offsets it per launch group)
    a.root_seq = seq;
    return merkle_batch_launches(
        a, (long long)batch, [&](int trees) { return get_tickets(st, trees); }, shape_spec,
        [&](MerkleArgs &m, int trees, bool last) -> int {
            MerkleArgs k = m;
            if (!last) k.root_out = nullptr;  // only the launch that finishes the trees publishes
            k_merkle_chunk<<<dim3((unsigned)(k.width / k.chunk), (unsigned)trees), MK_THREADS, 0, st>>>(k);
            SA_LAUNCH_CHECK();
            return SA_OK;
        });
}

extern "C" {

int sa_merkle_tree_batch(void *trees, const void *values, size_t n, size_t batch, void *stream) {
    if (!host_is_pow2(n)) return SA_ENOTPOW2;
    if (batch == 0) return SA_OK;
    MerkleArgs a;
    memset(&a, 0, sizeof(a));
    a.tree = (uint64_t *)trees;
    a.tree_stride = 16 * (long long)n;
    a.row_stride = (long long)n;
    a.width = (long long)n;
    a.mode = 1;
    a.values = (const fe *)values;
    return merkle_reduce(a, batch, (cudaStream_t)stream);
}

int sa_merkle_tree(void *tree, const void *values, size_t n, void *stream) {
    return sa_merkle_tree_batch(tree, values, n, 1, stream);
}

// checks the index sets (index_sets_check) and, when the call has work (`work`, k > 0), uploads them to
// stream-ordered device memory; *idx stays nullptr otherwise
static int upload_indices(uint64_t **idx, const uint64_t *indices_host, size_t batch, size_t group, size_t k, size_t n,
                          bool work, cudaStream_t st) {
    size_t count = 0;
    SA_TRY(index_sets_check(indices_host, batch, group, k, n, &count));
    *idx = nullptr;
    if (!work || count == 0) return SA_OK;
    keep_pool_memory();
    SA_CUDA(cudaMallocAsync((void **)idx, 8 * count, st));
    SA_CUDA(cudaMemcpyAsync(*idx, indices_host, 8 * count, cudaMemcpyHostToDevice, st));
    return SA_OK;
}

int sa_merkle_open_batch_sets(void *paths_out, const void *trees, size_t n, size_t batch, size_t group,
                              const uint64_t *indices_host, size_t k, void *stream) {
    if (!host_is_pow2(n)) return SA_ENOTPOW2;
    const int depth = host_log2(n);
    cudaStream_t st = (cudaStream_t)stream;
    uint64_t *idx = nullptr;
    int rc = upload_indices(&idx, indices_host, batch, group, k, n, batch != 0 && depth != 0, st);
    if (rc != SA_OK || idx == nullptr) return rc;
    const long long total = (long long)batch * (long long)k * depth * 8;
    k_merkle_paths<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((uint64_t *)paths_out,
                                                                    (const uint64_t *)trees, (long long)n,
                                                                    depth, idx, (long long)k, (long long)batch,
                                                                    (long long)group);
    SA_LAUNCH_CHECK();
    cudaFreeAsync(idx, st);
    return SA_OK;
}

int sa_merkle_open_batch(void *paths_out, const void *trees, size_t n, size_t batch, const uint64_t *indices_host,
                         size_t k, void *stream) {
    return sa_merkle_open_batch_sets(paths_out, trees, n, batch, batch ? batch : 1, indices_host, k, stream);
}

int sa_merkle_open(void *paths_out, const void *tree, size_t n, const uint64_t *indices_host, size_t k,
                   void *stream) {
    return sa_merkle_open_batch(paths_out, tree, n, 1, indices_host, k, stream);
}

int sa_gather_batch_sets(void *out, const void *values, size_t n, size_t batch, size_t group,
                         const uint64_t *indices_host, size_t k, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    uint64_t *idx = nullptr;
    int rc = upload_indices(&idx, indices_host, batch, group, k, n, batch != 0, st);
    if (rc != SA_OK || idx == nullptr) return rc;
    const long long total = (long long)batch * (long long)k;
    k_gather<<<(unsigned)((total + 127) / 128), 128, 0, st>>>((fe *)out, (const fe *)values, (long long)n, idx,
                                                            (long long)k, (long long)batch, (long long)group);
    SA_LAUNCH_CHECK();
    cudaFreeAsync(idx, st);
    return SA_OK;
}

int sa_gather_batch(void *out, const void *values, size_t n, size_t batch, const uint64_t *indices_host, size_t k,
                    void *stream) {
    return sa_gather_batch_sets(out, values, n, batch, batch ? batch : 1, indices_host, k, stream);
}

int sa_gather(void *out, const void *values, size_t n, const uint64_t *indices_host, size_t k, void *stream) {
    return sa_gather_batch(out, values, n, 1, indices_host, k, stream);
}

// x_i^-1 tables: xinv[i] = omega^-i (Montgomery), i < n/2, cached per (device, omega, n) in the LRU above
static int get_xinv(XinvPtr *out, const fe &omega, size_t n, cudaStream_t st) {
    int dev = 0;
    SA_CUDA(cudaGetDevice(&dev));
    const CacheKey key(1, dev, (uint64_t)n, (uint64_t)omega.v[0] | ((uint64_t)omega.v[1] << 32),
                       (uint64_t)omega.v[2] | ((uint64_t)omega.v[3] << 32), 0);
    if ((*out = cache_find<XinvTable>(key))) return SA_OK;
    const fe winv_m = fe_mont_inv(fe_to_mont(omega));
    XinvPtr made = std::make_shared<XinvTable>();
    made->device = dev;
    int rc = build_pow_table(*made, &made->tab, winv_m, fe_mont_one(), (long long)(n / 2), st);
    if (rc != SA_OK) return rc;
    SA_CUDA(cudaStreamSynchronize(st));  // complete before other streams can find it in the cache
    *out = cache_publish<XinvTable>(key, made);
    return SA_OK;
}

int sa_fri_fold(void *next, const void *cw, size_t n, const uint64_t alpha[2], const uint64_t offset[2],
                const uint64_t omega[2], void *stream) {
    if (!host_is_pow2(n) || n < 2) return SA_ENOTPOW2;
    cudaStream_t st = (cudaStream_t)stream;
    XinvPtr xinv;
    int rc = get_xinv(&xinv, fe_from_limbs(omega), n, st);
    if (rc != SA_OK) return rc;
    fe s_m, inv2_m;
    fri_fold_scalars(&s_m, &inv2_m, fe_from_limbs(alpha), fe_mont_inv(fe_to_mont(fe_from_limbs(offset))));
    k_fri_fold<<<grid_for((long long)(n / 2), 128), 128, 0, st>>>((fe *)next, (const fe *)cw,
                                                                 (long long)(n / 2), xinv->tab, s_m, inv2_m);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

int sa_fri_round(void *next, void *next_tree, const void *cw, size_t n, const uint64_t alpha[2],
                 const uint64_t offset[2], const uint64_t omega[2], void *stream) {
    if (!host_is_pow2(n) || n < 2) return SA_ENOTPOW2;
    cudaStream_t st = (cudaStream_t)stream;
    XinvPtr xinv;
    int rc = get_xinv(&xinv, fe_from_limbs(omega), n, st);
    if (rc != SA_OK) return rc;
    SA_CUDA(cudaMemsetAsync(next_tree, 0, 64, st));
    MerkleArgs a;
    memset(&a, 0, sizeof(a));
    a.tree = (uint64_t *)next_tree;
    a.width = (long long)(n / 2);
    a.mode = 2;
    a.prev = (const fe *)cw;
    a.next = (fe *)next;
    a.xinv = xinv->tab;
    fri_fold_scalars(&a.s_m, &a.inv2_m, fe_from_limbs(alpha), fe_mont_inv(fe_to_mont(fe_from_limbs(offset))));
    return merkle_reduce(a, 1, st);
}

// spin until the kernel has published root number `seq` (see merkle_publish_root); the stream is
// polled now and then so that a failed launch turns into an error instead of a hang
static int wait_for_root(uint64_t *root_host, unsigned long long seq, cudaStream_t st) {
    volatile uint64_t *flag = root_host + 8;
    for (unsigned spins = 1; *flag != seq; spins++) {
        if ((spins & 0xfff) == 0) {
            const cudaError_t q = cudaStreamQuery(st);
            if (q == cudaSuccess) {
                if (*flag == seq) break;
                g_last_error = "sa_fri_commit: the stream drained without publishing the round root";
                return SA_ECUDA;
            }
            if (q != cudaErrorNotReady) {
                g_last_error = std::string("sa_fri_commit: ") + cudaGetErrorString(q);
                return SA_ECUDA;
            }
        }
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    return SA_OK;
}

int sa_fri_commit(void *layers, void *trees, const void *codeword, size_t n, int rounds,
                  const uint64_t offset[2], const uint64_t omega[2], sa_fri_challenge_fn challenge, void *user,
                  void *stream) {
    if (!host_is_pow2(n) || rounds < 1 || (n >> (rounds - 1)) < 1) return SA_ESIZE;
    cudaStream_t st = (cudaStream_t)stream;
    // landing pad of the per-round root: words 0..7 the root, word 8 its sequence number, written by the
    // kernel itself (merkle_publish_root)
    static thread_local uint64_t *root_pinned = nullptr;
    static thread_local uint64_t *root_dev = nullptr;  // the same memory as the device addresses it
    static thread_local unsigned long long root_seq = 0;
    if (!root_pinned) {
        SA_CUDA(cudaHostAlloc((void **)&root_pinned, 256, cudaHostAllocMapped | cudaHostAllocPortable));
        memset(root_pinned, 0, 256);
    }
    SA_CUDA(cudaHostGetDevicePointer((void **)&root_dev, root_pinned, 0));  // per current device
    fe off = fe_from_limbs(offset), om = fe_from_limbs(omega);
    // offset^-1 is inverted once and then squared along with offset (fri_fold_scalars)
    fe oinv_m = fe_mont_inv(fe_to_mont(off));
    const fe *cur = (const fe *)codeword;
    fe *layer_out = (fe *)layers;
    uint8_t *tree = (uint8_t *)trees;
    size_t len = n;
    int rc;
    static const bool trace = getenv("SA_FRI_TRACE") != nullptr;  // per-round host timeline on stderr
    auto now = [] { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    double t_mark = now();
    for (int r = 0; r < rounds; r++) {
        if (r == 0) {
            MerkleArgs a;
            memset(&a, 0, sizeof(a));
            a.tree = (uint64_t *)tree;
            a.width = (long long)len;
            a.mode = 1;
            a.values = cur;
            if ((rc = merkle_reduce(a, 1, st, root_dev, ++root_seq)) != SA_OK) return rc;
        }
        const double t_launched = now();
        if ((rc = wait_for_root(root_pinned, root_seq, st)) != SA_OK) return rc;
        const double t_synced = now();
        uint64_t alpha[2] = {0, 0};
        const int want = r != rounds - 1;
        if (challenge(user, r, (const uint8_t *)root_pinned, alpha, want) != 0) return SA_ECALLBACK;
        if (trace) {
            const double t_cb = now();
            fprintf(stderr, "sa_fri_commit round %2d len %8zu: launch %.1f us, wait %.1f us, callback %.1f us\n", r, len,
                    t_launched - t_mark, t_synced - t_launched, t_cb - t_synced);
            t_mark = t_cb;
        }
        if (!want) break;
        // fold layer r into layer r+1 and build its tree
        uint8_t *next_tree = tree + 128 * len;  // this tree has 2 * len nodes of 64 bytes
        XinvPtr xinv;
        if ((rc = get_xinv(&xinv, om, len, st)) != SA_OK) return rc;
        MerkleArgs a;
        memset(&a, 0, sizeof(a));
        a.tree = (uint64_t *)next_tree;
        a.width = (long long)(len / 2);
        a.mode = 2;
        a.prev = cur;
        a.next = layer_out;
        a.xinv = xinv->tab;
        fri_fold_scalars(&a.s_m, &a.inv2_m, fe_from_limbs(alpha), oinv_m);
        if ((rc = merkle_reduce(a, 1, st, root_dev, ++root_seq)) != SA_OK) return rc;
        cur = layer_out;
        layer_out += len / 2;
        tree = next_tree;
        len /= 2;
        const fe om_m = fe_to_mont(om), off_m = fe_to_mont(off);
        om = fe_montmul(om_m, om);      // omega^2  (Montgomery form times canonical = canonical product)
        off = fe_montmul(off_m, off);   // offset^2
        oinv_m = fe_montmul(oinv_m, oinv_m);  // (offset^2)^-1, stays in Montgomery form
    }
    return SA_OK;
}

// what sa_fri_commit_batch keeps between calls of a thread: pinned, mapped host memory holding the landing pads of
// a round's roots (9 words per tree, merkle_publish_root) and then every round's fold scalars, which each round
// copies to the device in stream order
struct FriBatchHost {
    uint64_t *pinned = nullptr;
    size_t bytes = 0;
    unsigned long long seq = 0;  // the sequence number of the last round published
};

int sa_fri_commit_batch(void *layers, void *trees, const void *codewords, size_t n, size_t batch, int rounds,
                        const uint64_t offset[2], const uint64_t omega[2], sa_fri_challenge_batch_fn challenge,
                        void *user, void *stream) {
    SA_TRY(fri_commit_batch_check(layers, trees, codewords, n, batch, rounds, offset, omega, (const void *)challenge));
    if (batch == 0) return SA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    static thread_local FriBatchHost host;
    const size_t pad_words = 9 * batch, need = 8 * pad_words + sizeof(fe) * batch * (size_t)(rounds - 1);
    if (host.bytes < need) {
        if (host.pinned) {
            SA_CUDA(cudaFreeHost(host.pinned));
            host = FriBatchHost{nullptr, 0, host.seq};
        }
        SA_CUDA(cudaHostAlloc((void **)&host.pinned, need, cudaHostAllocMapped | cudaHostAllocPortable));
        memset(host.pinned, 0, need);  // no sequence number is 0
        host.bytes = need;
    }
    uint64_t *pad_dev = nullptr;
    SA_CUDA(cudaHostGetDevicePointer((void **)&pad_dev, host.pinned, 0));  // per current device
    fe *s_host = (fe *)(host.pinned + pad_words);
    fe *s_dev = nullptr;  // every round's scalars, freed in stream order whatever the outcome
    if (rounds > 1) {
        keep_pool_memory();
        SA_CUDA(cudaMallocAsync((void **)&s_dev, sizeof(fe) * batch * (size_t)(rounds - 1), st));
    }
    struct Free {
        fe *p;
        cudaStream_t st;
        ~Free() {
            if (p) cudaFreeAsync(p, st);
        }
    } free_s{s_dev, st};
    const long long B = (long long)batch;
    XinvPtr xinv;  // keeps the current round's table alive
    struct Ops {
        long long B;
        cudaStream_t st;
        uint64_t *pad_host, *pad_dev;
        unsigned long long &seq;
        fe *s_host, *s_dev;
        XinvPtr &tab;
        sa_fri_challenge_batch_fn fn;
        void *user;
        int tree(const MerkleArgs &a, int) { return merkle_reduce(a, (size_t)B, st, pad_dev, ++seq); }
        int roots(int, uint8_t *out) {
            for (long long b = 0; b < B; b++) {  // the one wait of the round: every tree's sequence word
                SA_TRY(wait_for_root(pad_host + 9 * b, seq, st));
                memcpy(out + 64 * b, pad_host + 9 * b, 64);
            }
            return SA_OK;
        }
        int challenge(int r, const uint8_t *roots, uint64_t *alphas, int want) { return fn(user, r, roots, alphas, want); }
        int xinv(const fe **out, const fe &omega, long long len) {
            SA_TRY(get_xinv(&tab, omega, (size_t)len, st));
            *out = tab->tab;
            return SA_OK;
        }
        int scalars(const fe **dev, int r, const fe *host) {
            fe *h = s_host + (size_t)r * B, *d = s_dev + (size_t)r * B;
            memcpy(h, host, sizeof(fe) * B);
            SA_CUDA(cudaMemcpyAsync(d, h, sizeof(fe) * B, cudaMemcpyHostToDevice, st));
            *dev = d;
            return SA_OK;
        }
    };
    return fri_commit_batch_rounds(Ops{B, st, host.pinned, pad_dev, host.seq, s_host, s_dev, xinv, challenge, user},
                                   (fe *)layers, (uint64_t *)trees, (const fe *)codewords, (long long)n, B, rounds,
                                   fe_from_limbs(offset), fe_from_limbs(omega));
}

}  // extern "C"
