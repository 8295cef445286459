// tests/emu/emu.cpp -- TEST INFRASTRUCTURE: runs the kernels' __host__ __device__
// phase functions (stark-anatomy_b200/csrc/*.cuh) on the CPU, thread by thread and
// barrier phase by barrier phase, so the index maps, twiddle tables and the
// portable field arithmetic can be checked against the oracle without a GPU.
// The host-side schedule around them (NTT plan and passes, Merkle launch loop,
// fold scalars, the subproduct tree's levels, walk, plan build and up-sweep) is
// the library's own, from the same headers; only the launches are replaced by
// CPU loops.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu.so emu.cpp
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../stark-anatomy_b200/csrc/field.cuh"
#include "../../stark-anatomy_b200/csrc/fri_merkle.cuh"
#include "../../stark-anatomy_b200/csrc/hash.cuh"
#include "../../stark-anatomy_b200/csrc/ntt_plan.cuh"
#include "../../stark-anatomy_b200/csrc/ntt_tile.cuh"
#include "../../stark-anatomy_b200/csrc/poly_tree.cuh"

using namespace sa;

static int g_elog = 4, g_c = 8;  // tile shape under test (emu_set_shape)

template <int LOGL, int ELOG, int C, int FLAGS>
static void run_tiles_variant(const TileArgs &a) {
    using P = TilePlan<LOGL, ELOG, C>;
    using S = TileStages<LOGL, ELOG, C, FLAGS>;
    const int tiles_per_batch = (a.ncols + C - 1) / C;
    const long long total = (long long)tiles_per_batch * a.nbatch;
    std::vector<fe> sm((size_t)P::L * C);
    for (long long tile = 0; tile < total; tile++) {
        const long long b = tile / tiles_per_batch;
        const int col0 = (int)(tile % tiles_per_batch) * C;
        // each loop over t is one barrier phase of the CTA
        for (int st = 0; st < P::NLOOP; st++)
            for (int t = 0; t < P::TPT; t++) S::full(st, t, sm.data(), a, b, col0, true, a.tw, nullptr);
        for (int t = 0; t < P::TPT; t++) S::last(t, sm.data(), a, b, col0, true);
    }
}
template <int LOGL, int ELOG, int C>
static void run_tiles(const TileArgs &a) {  // same variant choice as launch_tile (ntt.cu)
    if constexpr (LOGL >= 5) {
        switch (tile_variant<LOGL, ELOG, C>(a)) {
            case TF_FULL | TF_TWB: return run_tiles_variant<LOGL, ELOG, C, TF_FULL | TF_TWB>(a);
            case TF_FULL: return run_tiles_variant<LOGL, ELOG, C, TF_FULL>(a);
        }
    }
    return run_tiles_variant<LOGL, ELOG, C, TF_DYNAMIC>(a);
}
template <int LOGL>
static void run_tiles_shape(const TileArgs &a) {
    if (g_elog == 3 && g_c == 8) return run_tiles<LOGL, 3, 8>(a);
    if (g_elog == 3 && g_c == 4) return run_tiles<LOGL, 3, 4>(a);
    if (g_elog == 3 && g_c == 2) return run_tiles<LOGL, 3, 2>(a);
    if (g_elog == 4 && g_c == 4) return run_tiles<LOGL, 4, 4>(a);
    if (g_elog == 4 && g_c == 2) return run_tiles<LOGL, 4, 2>(a);
    if (g_elog == 4 && g_c == 3) return run_tiles<LOGL, 4, 3>(a);  // another non-power-of-two width (48-byte rows)
    if (g_elog == 4 && g_c == 7) return run_tiles<LOGL, 4, 7>(a);  // a non-power-of-two width (ragged: 1024 = 146 * 7 + 2)
    return run_tiles<LOGL, 4, 8>(a);
}
static void run_tiles_dyn(int logl, const TileArgs &a) {
    switch (logl) {
        case 1: run_tiles_shape<1>(a); break;
        case 2: run_tiles_shape<2>(a); break;
        case 3: run_tiles_shape<3>(a); break;
        case 4: run_tiles_shape<4>(a); break;
        case 5: run_tiles_shape<5>(a); break;
        case 6: run_tiles_shape<6>(a); break;
        case 7: run_tiles_shape<7>(a); break;
        case 8: run_tiles_shape<8>(a); break;
        case 9: run_tiles_shape<9>(a); break;
        case 10: run_tiles_shape<10>(a); break;
    }
}
// the tables of k_pow_table / k_twb_table, thread by thread
static std::vector<fe> pow_table(const fe &base_m, long long count, int swz) {
    std::vector<fe> t((size_t)count);
    for (long long i = 0; i < (count + 15) / 16; i++) ntt_pow_table_thread(t.data(), base_m, fe_mont_one(), count, swz, i);
    return t;
}
static std::vector<fe> twb_table(const fe &w_m, const fe &scale_m, int rows, long long cols) {
    std::vector<fe> t((size_t)rows * cols);
    for (long long i = 0; i < rows * ((cols + 15) / 16); i++)
        ntt_twb_table_thread(t.data(), w_m, scale_m, rows, (int)cols, i);
    return t;
}

extern "C" {

void emu_set_shape(int elog, int c) {
    g_elog = elog;
    g_c = c;
}

void emu_montmul(uint64_t *out, const uint64_t *a, const uint64_t *b) {
    fe r = fe_montmul_portable(fe_from_limbs(a), fe_from_limbs(b));
    memcpy(out, &r, 16);
}
void emu_mul(uint64_t *out, const uint64_t *a, const uint64_t *b) {
    fe r = fe_mul(fe_from_limbs(a), fe_from_limbs(b));
    memcpy(out, &r, 16);
}
void emu_add(uint64_t *out, const uint64_t *a, const uint64_t *b) {
    fe r = fe_add_portable(fe_from_limbs(a), fe_from_limbs(b));
    memcpy(out, &r, 16);
}
void emu_sub(uint64_t *out, const uint64_t *a, const uint64_t *b) {
    fe r = fe_sub_portable(fe_from_limbs(a), fe_from_limbs(b));
    memcpy(out, &r, 16);
}
void emu_inv(uint64_t *out, const uint64_t *a) {
    fe r = fe_from_mont(fe_mont_inv(fe_to_mont(fe_from_limbs(a))));
    memcpy(out, &r, 16);
}

// sa_ntt: the library's plan and pass sequence (ntt_plan.cuh) over the emulated tile passes.  force3 != 0
// uses the three-pass split (normally only for log_n > 20) so that it can be exercised at small sizes.
int emu_ntt_ex(uint64_t *out, const uint64_t *in, int log_n, const uint64_t *root, int inverse, size_t batch,
               int force3) {
    const size_t n = size_t(1) << log_n;
    if (log_n == 0) {
        memcpy(out, in, 16 * batch);
        return 0;
    }
    const fe root_m = fe_to_mont(fe_from_limbs(root));
    int rc = ntt_check_root(root_m, log_n);
    if (rc != SA_OK) return rc;
    const NttShape s = ntt_shape(log_n, force3 != 0);
    std::vector<std::vector<fe>> tables;
    NttTables t;
    auto keep = [&](fe **table, std::vector<fe> v) {
        tables.push_back(std::move(v));
        *table = tables.back().data();
        return SA_OK;
    };
    ntt_build_tables(
        t, s, root_m, inverse, [&](fe **table, const fe &base_m, long long count) { return keep(table, pow_table(base_m, count, 1)); },
        [&](fe **table, const fe &w_m, const fe &scale_m, int rows, long long cols) {
            return keep(table, twb_table(w_m, scale_m, rows, cols));
        });
    // the threads of a tile run one after another here, so a single pass in place would overwrite input
    // that later threads still read: it reads a copy
    std::vector<fe> tmp(n * batch);
    const fe *src = (const fe *)in;
    if (s.l2 == 0) src = (const fe *)memcpy(tmp.data(), in, 16 * n * batch);
    return ntt_run_passes(s, t, src, (fe *)out, tmp.data(), batch, [](int logl, TileArgs &a, bool) {
        run_tiles_dyn(logl, a);
        return SA_OK;
    });
}
int emu_ntt(uint64_t *out, const uint64_t *in, int log_n, const uint64_t *root, int inverse, size_t batch) {
    return emu_ntt_ex(out, in, log_n, root, inverse, batch, 0);
}

}  // extern "C"

// the backend of the subproduct tree's schedule (poly_tree.cuh): every kernel is a loop over its element function,
// sa_ntt is emu_ntt, device memory is host memory
struct EmuTree {
    template <class F>
    static int each(long long n, F f) {
        for (long long i = 0; i < n; i++) f(i);
        return SA_OK;
    }
    int leaves(fe *v0, const fe *d, long long k, long long K) {
        return each(K, [&](long long i) { tree_leaves_elem(v0, d, k, i); });
    }
    int pad(fe *dst, const fe *src, long long K, int mlog) {
        return each(2 * K, [&](long long i) { tree_pad_elem(dst, src, mlog, i); });
    }
    int pairmul(fe *out, const fe *in, long long K, int mlog) {
        return each(K, [&](long long i) { tree_pairmul_elem(out, in, mlog, i); });
    }
    int cross(fe *out, const fe *Pt, const fe *Vt, long long K, long long batch, int mlog) {
        return each(batch * K, [&](long long i) { tree_cross_elem(out, Pt, Vt, K, mlog, i); });
    }
    int fix(fe *parent, const fe *add, long long K, long long batch, int mlog, long long k) {
        return each(batch * K / 2, [&](long long i) { tree_fix_elem(parent, add, K, mlog, k, i); });
    }
    int derivative(fe *out, const fe *z, long long k) {
        return each(k, [&](long long i) { derivative_elem(out, z, i); });
    }
    int qleaves(fe *P0, const fe *values, const fe *inv_m, long long k, int logK, long long batch) {
        return each(batch << logK, [&](long long i) { tree_qleaves_elem(P0, values, inv_m, k, logK, i); });
    }
    int root(fe *out, const fe *root, long long k, long long K) {
        return each(k + 1, [&](long long i) { tree_root_elem(out, root, K, i); });
    }
    int series_pad(fe *W, const fe *z, long long k, const fe *alpha, long long s) {
        return each(8 * s, [&](long long i) { series_pad_elem(W, z, k, alpha, s, i); });
    }
    int series_step(fe *W, long long n4) {
        return each(n4, [&](long long i) { series_step_elem(W, n4, i); });
    }
    int eval_top_pad(fe *W, const fe *f, long long nf, const fe *alpha, long long n, long long n2) {
        return each(2 * n2, [&](long long i) { eval_top_pad_elem(W, f, nf, alpha, n, n2, i); });
    }
    int pointwise_mul(fe *out, const fe *a, const fe *b, long long n) {
        return each(n, [&](long long i) { pointwise_mul_elem(out, a, b, i); });
    }
    int eval_root(fe *c, const fe *s, long long n, long long k, long long K) {
        return each(K, [&](long long i) { eval_root_elem(c, s, n, k, i); });
    }
    int down(fe *O, const fe *chat, const fe *VT, long long K, int mlog) {
        return each(2 * K, [&](long long i) { tree_down_elem(O, chat, VT, mlog, i); });
    }
    int down_fix(fe *next, const fe *O, const fe *cur, long long K, int mlog, long long k) {
        return each(K, [&](long long i) { tree_down_fix_elem(next, O, cur, mlog, k, i); });
    }
    // one group of 8 consecutive elements per thread: the inverses do not depend on the grouping
    int batch_inverse(fe *inv_m, const fe *b, long long n, int *flag) {
        return each((n + 7) / 8, [&](long long g) {
            batch_inverse_group(b, n, 8 * g, 1, flag, [&](long long i, const fe &x) { inv_m[i] = x; });
        });
    }
    int horner(fe *out, const fe *coeffs, long long ncoef, const fe *points, long long npoints) {
        return each(npoints, [&](long long j) { out[j] = poly_horner(coeffs, ncoef, points[j]); });
    }
    int ntt(fe *out, const fe *in, int log_n, const uint64_t root[2], int inverse, size_t batch) {
        return emu_ntt((uint64_t *)out, (const uint64_t *)in, log_n, root, inverse, batch);
    }
    int copy(fe *dst, const fe *src, size_t n) {
        memmove(dst, src, sizeof(fe) * n);
        return SA_OK;
    }
    int copy2d(fe *dst, size_t dpitch, const fe *src, size_t spitch, size_t width, size_t rows) {
        for (size_t r = 0; r < rows; r++) memmove(dst + r * dpitch, src + r * spitch, sizeof(fe) * width);
        return SA_OK;
    }
    int store(fe *dst, const fe &v) {
        *dst = v;
        return SA_OK;
    }
};

extern "C" {

// the library's tree schedules over EmuTree, at any k >= 1 (the library takes its direct kernels at small k)
int emu_zerofier(uint64_t *out, const uint64_t *domain, size_t k) {
    Tree t = tree_layout(k, TREE_ZEROFIER, 0);
    std::vector<fe> ws(t.elems);
    t.ws = ws.data();
    EmuTree b;
    return tree_zerofier(b, t, (fe *)out, (const fe *)domain);
}
// sa_poly_eval_mode 2: the walk down the tree; ncoef >= 1
int emu_poly_eval_walk(uint64_t *out, const uint64_t *coeffs, size_t ncoef, const uint64_t *points, size_t npoints) {
    Tree t = tree_layout(npoints, TREE_EVAL, ncoef);
    std::vector<fe> ws(t.elems);
    t.ws = ws.data();
    EmuTree b;
    return tree_poly_eval(b, t, (fe *)out, (const fe *)coeffs, ncoef, (const fe *)points);
}
size_t emu_interp_plan_bytes(size_t k) { return sizeof(fe) * interp_plan_layout(k, true).elems; }
// sa_interp_plan with the tree's layout; walk != 0: M'(d_i) by the walk down the tree, else by Horner
int emu_interp_plan(uint64_t *plan, const uint64_t *domain, size_t k, int walk) {
    const InterpPlan L = interp_plan_layout(k, true);
    if (L.elems == 0) return SA_ESIZE;
    Tree t = tree_layout(k, TREE_PLAN, walk ? k : 0);
    std::vector<fe> ws(t.elems);
    t.ws = ws.data();
    int flag = 0;
    EmuTree b;
    const int rc = interp_plan_tree(b, t, (fe *)plan, L, (const fe *)domain, walk != 0, &flag);
    return rc != SA_OK ? rc : flag ? SA_EDIVZERO : SA_OK;
}
int emu_interp_apply_batch(uint64_t *out, const uint64_t *plan, const uint64_t *values, size_t k, size_t batch) {
    const InterpPlan L = interp_plan_layout(k, true);
    if (L.elems == 0) return SA_ESIZE;
    std::vector<fe> ws(4 * (size_t)L.K * std::min(batch, interp_batch_max(L)));
    EmuTree b;
    return interp_apply_tree(b, (fe *)out, (const fe *)plan, L, (const fe *)values, k, batch, ws.data());
}

uint32_t emu_decimal(uint8_t *buf40, const uint64_t *x) {
    uint64_t w[5];
    uint32_t n = fe_decimal_words(w, fe_from_limbs(x));
    memcpy(buf40, w, 40);
    return n;
}
void emu_leaf_digest(uint8_t *out64, const uint64_t *x) {
    uint64_t d[8];
    merkle_leaf_digest(d, fe_from_limbs(x));
    memcpy(out64, d, 64);
}
void emu_node_digest_coop4(uint8_t *out64, const uint8_t *left, const uint8_t *right) {
    uint64_t m[16], d[8];
    memcpy(m, left, 64);
    memcpy(m + 8, right, 64);
    blake2b_coop4_node_host(d, m);
    memcpy(out64, d, 64);
}
void emu_node_digest(uint8_t *out64, const uint8_t *left, const uint8_t *right) {
    uint64_t l[8], r[8], d[8];
    memcpy(l, left, 64);
    memcpy(r, right, 64);
    merkle_node_digest(d, l, r);
    memcpy(out64, d, 64);
}

// one launch of k_merkle_chunk without the fused top: private subtrees, then the shared-memory reduction
static int emu_merkle_chunk(const MerkleArgs &a) {
    std::vector<uint64_t> sm((size_t)MK_THREADS * 8);
    const long long blocks = a.width / a.chunk;
    const int active = a.chunk >> a.ipt_log;
    for (long long blk = 0; blk < blocks; blk++) {
        for (int tid = 0; tid < active; tid++) merkle_private(&sm[(size_t)tid * 8], a, blk, tid);
        long long base = (a.width + blk * a.chunk) >> a.ipt_log;
        for (int wl = active / 2, lvl = 0; lvl < a.red_log; wl >>= 1, lvl++) {
            base >>= 1;
            std::vector<uint64_t> regs((size_t)wl * 8);
            for (int tid = 0; tid < wl; tid++) {  // phase 1: read children, hash
                if (wl > a.coop_max)
                    merkle_node_digest(&regs[(size_t)tid * 8], &sm[(size_t)(2 * tid) * 8],
                                       &sm[(size_t)(2 * tid + 1) * 8]);
                else  // the four-lanes-per-node schedule of the small levels
                    blake2b_coop4_node_host(&regs[(size_t)tid * 8], &sm[(size_t)(2 * tid) * 8]);
            }
            for (int tid = 0; tid < wl; tid++)  // phase 2: publish
                for (int i = 0; i < 8; i++) {
                    sm[(size_t)tid * 8 + i] = regs[(size_t)tid * 8 + i];
                    a.tree[(base + tid) * 8 + i] = regs[(size_t)tid * 8 + i];
                }
        }
    }
    return 0;
}
static std::string g_mk_shape;  // launch shape override in SA_MK_SHAPE form (tests try other launch shapes)
// the library's launch loop without an arrival counter, which the library falls back to without one
static void emu_merkle_reduce(const MerkleArgs &a) {
    merkle_launches(a, nullptr, g_mk_shape.c_str(), [](MerkleArgs &m, bool) { return emu_merkle_chunk(m); });
}
void emu_set_merkle_shape(const char *spec) { g_mk_shape = spec ? spec : ""; }
int emu_merkle_tree(uint8_t *tree, const uint64_t *values, size_t n) {
    memset(tree, 0, 64);
    MerkleArgs a;
    memset(&a, 0, sizeof(a));
    a.tree = (uint64_t *)tree;
    a.width = (long long)n;
    a.mode = 1;
    a.values = (const fe *)values;
    emu_merkle_reduce(a);
    return 0;
}
int emu_fri_round(uint64_t *next, uint8_t *next_tree, const uint64_t *cw, size_t n, const uint64_t *alpha,
                  const uint64_t *offset, const uint64_t *omega) {
    memset(next_tree, 0, 64);
    const fe winv_m = fe_mont_inv(fe_to_mont(fe_from_limbs(omega)));
    std::vector<fe> xinv = pow_table(winv_m, (long long)(n / 2), 0);
    MerkleArgs a;
    memset(&a, 0, sizeof(a));
    a.tree = (uint64_t *)next_tree;
    a.width = (long long)(n / 2);
    a.mode = 2;
    a.prev = (const fe *)cw;
    a.next = (fe *)next;
    a.xinv = xinv.data();
    fri_fold_scalars(&a.s_m, &a.inv2_m, fe_from_limbs(alpha), fe_mont_inv(fe_to_mont(fe_from_limbs(offset))));
    emu_merkle_reduce(a);
    return 0;
}

}  // extern "C"
