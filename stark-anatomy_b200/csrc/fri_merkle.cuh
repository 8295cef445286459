// fri_merkle.cuh -- per-thread pieces of the FRI round kernel: split-and-fold
// (code/fri.py:85) and the chunked Merkle reduction (code/merkle.py:6-14).
// __host__ __device__ so tests/emu can drive the same code phase by phase; the launch loop of a tree,
// the fold scalars and the round loop of the batched commit are shared with it too.
#pragma once
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

#include "field.cuh"
#include "hash.cuh"
#include "host.cuh"
#include "ntt_tile.cuh"

namespace sa {

constexpr int MK_THREADS = 256;  // threads per Merkle CTA
constexpr int MK_MAX_IPT_LOG = 3;  // a thread reduces at most 8 bottom nodes privately
constexpr int MK_MAX_TREES = 65535;  // trees per launch: the tree of a CTA is blockIdx.y

// c'[i] = 2^-1 (a + b) + (alpha * 2^-1 * x_i^-1) (a - b)   ==  fri.py:85
//   inv2_m : 2^-1 in Montgomery form
//   t_m    : alpha * 2^-1 * (offset * omega^i)^-1 in Montgomery form
SA_HD fe fri_fold_one(const fe &a, const fe &b, const fe &t_m, const fe &inv2_m) {
    const fe s = fe_montmul(fe_add(a, b), inv2_m);
    const fe d = fe_montmul(fe_sub(a, b), t_m);
    return fe_add(s, d);
}

SA_HD fe merkle_ld_stream(const fe *p) {
#if defined(__CUDA_ARCH__)
    const uint4 v = __ldcg(reinterpret_cast<const uint4 *>(p));
    return fe_make(v.x, v.y, v.z, v.w);
#else
    return *p;
#endif
}

struct MerkleArgs {
    uint64_t *tree;      // heap layout, 8 words per node; tree b of a batch at tree + b * tree_stride
    long long tree_stride;  // words from one tree of a batch to the next (16 per leaf), 0 without a batch
    long long row_stride;   // elements from one row of a batch to the next: mode 1 `values`, mode 2 `next`
                            // (mode 2 `prev` rows are twice as long)
    long long width;     // number of bottom nodes of this launch
    int chunk;           // bottom nodes per CTA (power of two, <= MK_THREADS << ipt_log)
    int ipt_log;         // log2 of the bottom nodes one thread reduces privately (0..3)
    int red_log;         // tree levels the CTA then reduces through shared memory (0..log2(chunk) - ipt_log);
                         // the launch leaves width >> (ipt_log + red_log) digests for the next one
    int coop_max;        // shared-memory levels of at most this many nodes are hashed four lanes per node
    int mode;            // 0: bottom digests already in tree; 1: leaves from `values`; 2: leaves from a fold
    const fe *values;    // mode 1: the codeword (width elements)
    const fe *prev;      // mode 2: the codeword being folded (2 * width elements)
    fe *next;            // mode 2: receives the folded codeword (width elements)
    const fe *xinv;      // mode 2: xinv[i] = omega^-i in Montgomery form, i < width
    fe s_m;              // mode 2: alpha * 2^-1 * offset^-1 in Montgomery form
    const fe *s_rows;    // mode 2, optional: tree b of a batch folds with s_rows[b] instead of s_m (device memory)
    fe inv2_m;           // mode 2: 2^-1 in Montgomery form
    unsigned int *ticket;  // optional: CTA arrival counters, one per tree (zero between launches); the CTA of a
                         // tree that arrives last also reduces its gridDim.x (<= MK_THREADS) subtree roots,
                         // saving a launch
    uint64_t *root_out;  // last launch of a tree, optional: host-mapped landing pad, receives the root (8 words)
    unsigned long long root_seq;  // and then this sequence number in word 8; tree b of a batch at root_out + 9 b
};

// the arguments of tree b of a batch: its nodes, its codeword rows, its fold scalar, its arrival counter and its
// landing pad (pointer arithmetic only: the host computes the views of a launch group)
SA_HD MerkleArgs merkle_view(const MerkleArgs &a, long long b) {
    MerkleArgs v = a;
    v.tree += b * a.tree_stride;
    v.values += b * a.row_stride;
    v.prev += 2 * b * a.row_stride;
    v.next += b * a.row_stride;
    if (v.s_rows) v.s_rows += b;
    if (v.ticket) v.ticket += b;
    if (v.root_out) v.root_out += 9 * b;
    return v;
}
// what the CTAs of tree b work with: its view, with its own fold scalar read once
SA_HD MerkleArgs merkle_tree_args(const MerkleArgs &a, long long b) {
    MerkleArgs v = merkle_view(a, b);
    if (v.s_rows) v.s_m = v.s_rows[0];
    return v;
}

// launch shape for a level of `width` bottom nodes: small levels are latency bound (one node per
// thread, 64..256-node CTAs so that 128-256 CTAs are in flight, each reducing its chunk to one digest); big ones are
// throughput bound: four leaves and their three parents per thread, barrier free, then only the three
// shared-memory levels that still fill whole warps (128, 64, 32 nodes) - the 32 digests a CTA leaves
// are picked up by the next launch, so no SM sits in a mostly idle dependency chain while thousands
// of leaves wait (tools/merkle_sweep.py times the shapes)
SA_HD int merkle_log2(long long x) {
    int l = 0;
    while ((1ll << l) < x) l++;
    return l;
}
SA_HD void merkle_shape(MerkleArgs &a) {
    a.coop_max = MK_THREADS / 4;  // latency bound: a level of <= 64 nodes keeps all 256 lanes busy that way
    a.ipt_log = 0;
    if (a.width <= 64) {  // one CTA finishes the tree
        a.chunk = (int)a.width;
    } else if (a.width < (1 << 14)) {
        // dependency-chain regime: few leaves per CTA spread the leaf hashes (a warp-wide compression
        // occupies its scheduler for the same time whatever the number of active lanes) over many SMs, and the CTA that arrives last reduces the <= 256
        // subtree roots, so the tree is still one launch
        a.chunk = 64;
    } else if (a.width < (1 << 15)) {
        a.chunk = 128;
    } else if (a.width < (1 << 16)) {
        a.chunk = MK_THREADS;
    } else if (a.width < (1 << 18)) {
        a.ipt_log = 1;
        a.chunk = MK_THREADS << 1;
    } else {  // throughput bound
        a.ipt_log = 2;
        a.chunk = MK_THREADS << 2;
        a.red_log = 3;
        a.coop_max = 0;  // one thread per node issues fewer instructions per node
        return;
    }
    a.red_log = merkle_log2(a.chunk) - a.ipt_log;  // each CTA reduces its chunk to one digest
}
// width of the level a launch of shape `a` leaves behind
SA_HD long long merkle_next_width(const MerkleArgs &a) { return a.width >> (a.ipt_log + a.red_log); }

// spec = "minlog:ipt:chunklog:red:coopmax,..." (SA_MK_SHAPE with -DSA_TUNE): the row with the largest
// minlog <= log2(width) (and chunklog <= log2(width)) replaces the launch shape of the level
inline void merkle_shape_override(MerkleArgs &a, const char *spec) {
    int best = -1, w = merkle_log2(a.width);
    while (*spec) {
        int ml, ipt, cl, red, coop, used = 0;
        if (sscanf(spec, "%d:%d:%d:%d:%d%n", &ml, &ipt, &cl, &red, &coop, &used) != 5) break;
        if (ml <= w && ml > best && cl <= w) {
            best = ml;
            a.ipt_log = ipt;
            a.chunk = 1 << cl;
            a.red_log = red;
            a.coop_max = coop;
        }
        spec += used;
        if (*spec == ',') spec++;
    }
}

// Launches of one tree: the first handles the bottom level in a.mode (and, in mode 1, zeroes the unused
// node 0), later ones continue from the digests the previous one left.  With an arrival counter (`ticket`), the launch that leaves at most
// MK_THREADS single-digest CTAs also reduces those; without one, that takes one more launch.
// shape_spec (nullptr: none) goes to merkle_shape_override.  launch(a, last) runs one launch and returns
// 0 or an error code; `last` marks the launch that finishes the tree.
template <class Launch>
int merkle_launches(MerkleArgs a, unsigned int *ticket, const char *shape_spec, Launch &&launch) {
    while (true) {
        merkle_shape(a);
        if (shape_spec) merkle_shape_override(a, shape_spec);
        const long long left = merkle_next_width(a), grid = a.width / a.chunk;
        const bool fuse_top = left > 1 && left <= MK_THREADS && left == grid && ticket != nullptr;
        const bool last = left <= 1 || fuse_top;
        a.ticket = fuse_top ? ticket : nullptr;
        const int rc = launch(a, last);
        if (rc != 0 || last) return rc;
        a.width = left;
        a.mode = 0;
    }
}

// Launches of `batch` trees of one width (merkle_view lays them out): groups of up to MK_MAX_TREES trees,
// each group issuing the launches of one tree.  tickets(trees) returns the arrival counters of a group
// (nullptr: none); launch(a, trees, last) runs one launch over the group's trees.
template <class Tickets, class Launch>
int merkle_batch_launches(const MerkleArgs &a, long long batch, Tickets &&tickets, const char *shape_spec,
                          Launch &&launch) {
    for (long long b0 = 0; b0 < batch; b0 += MK_MAX_TREES) {
        const int trees = (int)(batch - b0 < MK_MAX_TREES ? batch - b0 : MK_MAX_TREES);
        const int rc = merkle_launches(merkle_view(a, b0), tickets(trees), shape_spec,
                                       [&](MerkleArgs &m, bool last) { return launch(m, trees, last); });
        if (rc != 0) return rc;
    }
    return 0;
}

// the scalars of a fold (fri.py:85) in Montgomery form: inv2_m = 2^-1, s_m = alpha * 2^-1 * offset^-1.
// oinv_m is offset^-1 in Montgomery form: a commit squares it along with offset from round to round, since
// a Fermat inversion on the host costs ~10 us (a fifth of a round trip); 2^-1 is computed once.
inline void fri_fold_scalars(fe *s_m, fe *inv2_m, const fe &alpha, const fe &oinv_m) {
    static const fe inv2 = fe_mont_inv(fe_to_mont(fe_from_u64(2)));
    *inv2_m = inv2;
    *s_m = fe_montmul(fe_montmul(fe_to_mont(alpha), inv2), oinv_m);
}

// ---- the batched FRI commit (sa_fri_commit_batch): B codewords of one length, offset and omega ----
// Round r's B layers are back-to-back rows of n >> r elements (round 0's are the codewords), its B trees back-to-back
// heaps of 2 (n >> r) nodes, round after round.  Round 0 is one tree ladder over the B codewords, every later round
// one fused fold + tree ladder (mode 2) over the B rows of the previous round, each row folding with its own
// challenge.  ops supplies what the device and the emulation do differently:
//   ops.tree(a, r)                  the launches of round r's trees (merkle_batch_launches over the views of a)
//   ops.roots(r, out)               waits once for round r's B roots, 64 bytes each, into out
//   ops.challenge(r, roots, alphas, want)   the caller's callback: B alphas (two limbs each) when want
//   ops.xinv(&tab, omega, len)      xinv[i] = omega^-i in Montgomery form, i < len / 2
//   ops.scalars(&dev, r, host)      the B fold scalars of round r where the fold reads them
// Returns SA_OK, SA_ECALLBACK when the callback returns non-zero (nothing more is launched), or ops' error.
// sa_fri_commit_batch's refusals (SA_ESIZE); SA_OK for a batch of none whatever its buffers
inline int fri_commit_batch_check(const void *layers, const void *trees, const void *codewords, size_t n, size_t batch,
                                  int rounds, const void *offset, const void *omega, const void *challenge) {
    if (!host_is_pow2(n) || rounds < 1 || rounds - 1 > host_log2(n)) return SA_ESIZE;
    if (batch != 0 && (!trees || !codewords || (rounds > 1 && !layers) || !offset || !omega || !challenge))
        return SA_ESIZE;
    return SA_OK;
}
template <class Ops>
int fri_commit_batch_rounds(Ops &&ops, fe *layers, uint64_t *trees, const fe *codewords, long long n, long long batch,
                            int rounds, fe offset, fe omega) {
    std::vector<uint8_t> roots((size_t)(64 * batch));
    std::vector<uint64_t> alphas((size_t)(2 * batch));
    std::vector<fe> s((size_t)batch);
    fe oinv_m = fe_mont_inv(fe_to_mont(offset));  // squared along with offset (fri_fold_scalars)
    const fe *cur = codewords;
    long long len = n;
    MerkleArgs a;
    memset(&a, 0, sizeof(a));
    a.tree = trees;
    a.tree_stride = 16 * len;
    a.row_stride = len;
    a.width = len;
    a.mode = 1;
    a.values = cur;
    for (int r = 0;; r++) {
        SA_TRY(ops.tree(a, r));
        SA_TRY(ops.roots(r, roots.data()));
        const int want = r != rounds - 1;
        if (ops.challenge(r, (const uint8_t *)roots.data(), alphas.data(), want) != 0) return SA_ECALLBACK;
        if (!want) return SA_OK;
        const fe *xinv = nullptr;
        SA_TRY(ops.xinv(&xinv, omega, len));
        fe inv2_m;
        for (long long b = 0; b < batch; b++) fri_fold_scalars(&s[b], &inv2_m, fe_from_limbs(&alphas[2 * b]), oinv_m);
        const fe *s_rows = nullptr;
        SA_TRY(ops.scalars(&s_rows, r, s.data()));
        // fold round r's rows into round r + 1's and build their trees
        uint64_t *next_tree = a.tree + batch * 16 * len;
        fe *next = layers;
        layers += batch * (len / 2);
        memset(&a, 0, sizeof(a));
        a.tree = next_tree;
        a.tree_stride = 8 * len;
        a.row_stride = len / 2;
        a.width = len / 2;
        a.mode = 2;
        a.prev = cur;
        a.next = next;
        a.xinv = xinv;
        a.s_rows = s_rows;
        a.inv2_m = inv2_m;
        cur = next;
        len /= 2;
        omega = fe_montmul(fe_to_mont(omega), omega);  // omega^2 (Montgomery form times canonical = canonical)
        oinv_m = fe_montmul(oinv_m, oinv_m);           // (offset^2)^-1
    }
}

// digest of bottom node g of this launch: loads it (mode 0) or hashes the leaf (modes 1, 2) and
// writes it to the tree (and next[] in mode 2)
SA_HD void merkle_bottom(uint64_t d[8], const MerkleArgs &a, long long g) {
    uint64_t *node = a.tree + (a.width + g) * 8;
    if (a.mode == 0) {
        for (int i = 0; i < 8; i++) d[i] = node[i];
        return;
    }
    fe v;
    if (a.mode == 1) {
        v = a.values[g];
    } else {
        const fe t_m = fe_montmul(a.xinv[g], a.s_m);
        // (.cg: the layer is read exactly once, so caching it in L1 would gain nothing)
        v = fri_fold_one(merkle_ld_stream(a.prev + g), merkle_ld_stream(a.prev + a.width + g), t_m, a.inv2_m);
        a.next[g] = v;
    }
    merkle_leaf_digest(d, v);
    for (int i = 0; i < 8; i++) node[i] = d[i];
}

// Private phase of thread t of CTA blk: reduce its 2^ipt_log bottom nodes to one digest (streaming:
// a slot per height), writing every node it creates to the tree.  root = the subtree digest.
SA_HD void merkle_private(uint64_t root[8], const MerkleArgs &a, long long blk, int t) {
    uint64_t slot[MK_MAX_IPT_LOG][8];
    const int ipt = 1 << a.ipt_log;
    uint64_t d[8];
    for (int j = 0; j < ipt; j++) {
        const long long g = blk * a.chunk + (long long)t * ipt + j;
        merkle_bottom(d, a, g);
        long long idx = a.width + g;
        int h = 0;
        while ((j >> h) & 1) {  // a left sibling of this height is waiting: combine
            uint64_t l[8];
            for (int i = 0; i < 8; i++) l[i] = slot[h][i];
            merkle_node_digest(d, l, d);
            idx >>= 1;
            for (int i = 0; i < 8; i++) a.tree[idx * 8 + i] = d[i];
            h++;
        }
        if (h < a.ipt_log)
            for (int i = 0; i < 8; i++) slot[h][i] = d[i];
    }
    for (int i = 0; i < 8; i++) root[i] = d[i];
}

// ---- openings with an index set per group: sa_gather_batch_sets and sa_merkle_open_batch_sets ----
// Rows (trees) are taken in groups of `group`; row b reads set b / group, indices[(b / group) * k .. + k).  The
// ungrouped calls are group = batch: every row reads the one set.
// the number of indices the sets of a call hold, ceil(batch / group) sets of k and at least one (a call without rows
// still checks its indices), after checking them: SA_ESIZE for group == 0, SA_EINDEX for any index >= n
inline int index_sets_check(const uint64_t *indices, size_t batch, size_t group, size_t k, size_t n, size_t *count) {
    if (group == 0) return SA_ESIZE;
    *count = std::max<size_t>(1, (batch + group - 1) / group) * k;
    for (size_t i = 0; i < *count; i++)
        if (indices[i] >= n) return SA_EINDEX;
    return SA_OK;
}
// out[b][q] = values[b * n + the index q of row b's set]  (t = b * k + q < batch * k)
SA_HD void gather_sets_elem(fe *out, const fe *values, long long n, const uint64_t *indices, long long k,
                            long long group, long long t) {
    const long long b = t / k, q = t - b * k;
    tile_st(out + t, tile_ld(values + b * n + (long long)indices[(b / group) * k + q]));
}
// out[b][q][level] = word w of the sibling at `level` of the leaf index q of tree b's set, in tree b (trees 2n nodes
// apart)  (t = ((b * k + q) * depth + level) * 8 + w < batch * k * depth * 8)
SA_HD void merkle_path_sets_elem(uint64_t *out, const uint64_t *trees, long long n, int depth, const uint64_t *indices,
                                 long long k, long long group, long long t) {
    const int w = (int)(t & 7);
    const long long ql = t >> 3;
    const int level = (int)(ql % depth);
    const long long qb = ql / depth, q = qb % k, b = qb / k;
    const long long node = ((n + (long long)indices[(b / group) * k + q]) >> level) ^ 1;
    out[t] = trees[(b * 2 * n + node) * 8 + w];
}

}  // namespace sa
