// poly_tree.cuh -- the subproduct tree over k points (fast_zerofier / fast_evaluate / fast_interpolate,
// code/ntt.py:66-130): the per-element bodies of its kernels and the host schedule of every call that runs on it
// (the zerofier, the walk down, the tree half of an interpolation plan, the batched up-sweep).  The library
// (poly.cu) runs the schedule with kernel launches, the CPU emulation (tests/emu) with loops over the element
// functions.
//
// The schedule is instantiated with a backend B that has one method per kernel, named after it without the k_ /
// k_tree_ prefix (k_tree_pad -> b.pad, k_series_step -> b.series_step, k_poly_eval -> b.horner) and taking the
// kernel's arguments; b.ntt(out, in, log_n, root, inverse, batch) as sa_ntt; b.copy(dst, src, n),
// b.copy2d(dst, dpitch, src, spitch, width, rows) (in elements) and b.store(dst, v) (one element from the host).
// Every method returns SA_OK or an error code, and the schedule stops at the first error.
//
// The k points sit in the first k of K = 2^ceil(log2 k) leaf slots.  Level j has K >> j nodes of
// m = 2^j coefficients each, stored back to back.  A node whose leaf range lies completely inside the
// domain is FULL: its zerofier is monic of degree exactly m and only the low m coefficients are stored
// (the leading 1 is implied).  Any other node is stored EXPLICITLY (degree < m, all coefficients); a node
// without points is the constant 1.  With child vectors vL, vR a parent is
//     cyclic_product_2m(vL, vR) + x^m * ([L full] vR + [R full] vL)
// (the cyclic product of size 2m never wraps: both factors have degree < m), FULL iff both children are.
#pragma once
#include <algorithm>
#include <cstdint>
#include <mutex>

#include "host.cuh"
#include "ntt_tile.cuh"

namespace sa {

// ---- element functions: the body of each kernel for one index ----
SA_HD bool tree_full(long long node, int mlog, long long k) { return ((node + 1) << mlog) <= k; }
// leaf i: X - d_i, or the constant 1 for an empty slot (i < K)
SA_HD void tree_leaves_elem(fe *v0, const fe *domain, long long k, long long i) {
    tile_st(v0 + i, i < k ? fe_neg(tile_ld(domain + i)) : fe_one());
}
// dst node (2m slots) = [src node (m coefficients), m zeros]  (idx < 2K)
SA_HD void tree_pad_elem(fe *dst, const fe *src, int mlog, long long idx) {
    const long long m = 1ll << mlog, node = idx >> (mlog + 1), t = idx & (2 * m - 1);
    tile_st(dst + idx, t < m ? tile_ld(src + node * m + t) : fe_zero());
}
// transformed children (blocks of 2m) -> transformed parents: out[p][t] = in[2p][t] * in[2p+1][t]  (idx < K)
SA_HD void tree_pairmul_elem(fe *out, const fe *in, int mlog, long long idx) {
    const long long two_m = 2ll << mlog, p = idx >> (mlog + 1), t = idx & (two_m - 1);
    const fe a = tile_ld(in + (2 * p) * two_m + t), b = tile_ld(in + (2 * p + 1) * two_m + t);
    tile_st(out + idx, fe_montmul(fe_to_mont(a), b));
}
// interpolation up-sweep of trees of K slots, back to back, over one tree's node transforms Vt (2K):
// out[p][t] = P[2p][t] * V[2p+1][t] + P[2p+1][t] * V[2p][t]  (idx < batch * K)
SA_HD void tree_cross_elem(fe *out, const fe *Pt, const fe *Vt, long long K, int mlog, long long idx) {
    const long long two_m = 2ll << mlog, p = idx >> (mlog + 1), t = idx & (two_m - 1);
    const long long l = (2 * p) * two_m + t, r = (2 * p + 1) * two_m + t;
    const fe a = fe_montmul(fe_to_mont(tile_ld(Pt + l)), tile_ld(Vt + (r & (2 * K - 1))));
    const fe b = fe_montmul(fe_to_mont(tile_ld(Pt + r)), tile_ld(Vt + (l & (2 * K - 1))));
    tile_st(out + idx, fe_add(a, b));
}
// parent[p][m + t] += [L full] right[t] + [R full] left[t]; (left, right) = the child vectors of `add` (the
// zerofier tree adds the children's own vectors, the interpolation sweep the P vectors: P_L * M_R picks up
// x^m * P_L when M_R is full).  Trees of K slots, back to back: a node is full by its index within its own tree.
// (idx < batch * K / 2)
SA_HD void tree_fix_elem(fe *parent, const fe *add, long long K, int mlog, long long k, long long idx) {
    const long long m = 1ll << mlog, p = idx >> mlog, t = idx & (m - 1), left_node = (2 * p) & ((K >> mlog) - 1);
    const bool lfull = tree_full(left_node, mlog, k), rfull = tree_full(left_node + 1, mlog, k);
    if (!lfull && !rfull) return;
    const fe left = tile_ld(add + (2 * p) * m + t), right = tile_ld(add + (2 * p + 1) * m + t);
    fe acc = tile_ld(parent + p * 2 * m + m + t);
    if (lfull) acc = fe_add(acc, right);
    if (rfull) acc = fe_add(acc, left);
    tile_st(parent + p * 2 * m + m + t, acc);
}
// out[i] = (i + 1) * z[i + 1], i < k  (formal derivative of a polynomial with k + 1 coefficients)
SA_HD void derivative_elem(fe *out, const fe *z, long long i) {
    tile_st(out + i, fe_montmul(fe_to_mont(fe_from_u64((uint64_t)(i + 1))), tile_ld(z + i + 1)));
}
// leaves of the interpolation sweep: q_i = v_i / M'(d_i) for i < k (inv_m = the plan's Montgomery 1/M'(d_i)),
// 0 for the empty slots; vector b (values + b * k) fills the K = 2^logK slots at P0 + b * K  (idx < batch * K)
SA_HD void tree_qleaves_elem(fe *P0, const fe *values, const fe *inv_m, long long k, int logK, long long idx) {
    const long long b = idx >> logK, i = idx & ((1ll << logK) - 1);
    tile_st(P0 + idx, i < k ? fe_montmul(tile_ld(values + b * k + i), tile_ld(inv_m + i)) : fe_zero());
}
// zerofier coefficients from the tree's root vector: k == K -> implied leading 1  (i <= k)
SA_HD void tree_root_elem(fe *out, const fe *root, long long K, long long i) {
    tile_st(out + i, (i == K) ? fe_one() : tile_ld(root + i));
}
SA_HD void pointwise_mul_elem(fe *out, const fe *a, const fe *b, long long i) {
    tile_st(out + i, fe_montmul(fe_to_mont(tile_ld(a + i)), tile_ld(b + i)));
}
// Horner at one point (the coefficients are read through the read-only path, broadcast)
SA_HD fe poly_horner(const fe *coeffs, long long ncoef, const fe &x) {
    const fe x_m = fe_to_mont(x);
    fe acc = fe_zero();
    for (long long i = ncoef - 1; i >= 0; i--) acc = fe_add(fe_montmul(acc, x_m), tile_ldg(coeffs + i));
    return acc;
}
// Montgomery's batch-inversion trick over the 8 elements base + g * stride, g < 8 (one Fermat inverse for 8):
// emit(i, Montgomery form of 1/b[i]) for each of them below n; a zero b[i] raises *zero_flag and is inverted as 1
template <class Emit>
SA_HD void batch_inverse_group(const fe *b, long long n, long long base, long long stride, int *zero_flag, Emit emit) {
    constexpr int G = 8;
    fe bm[G], pre[G];
    fe acc = fe_mont_one();
#pragma unroll
    for (int g = 0; g < G; g++) {
        const long long i = base + g * stride;
        fe v = (i < n) ? tile_ld(b + i) : fe_one();
        if (fe_is_zero(v)) {
            *zero_flag = 1;
            v = fe_one();
        }
        bm[g] = fe_to_mont(v);
        pre[g] = acc;
        acc = fe_montmul(acc, bm[g]);
    }
    fe inv = fe_mont_inv(acc);
#pragma unroll
    for (int g = G - 1; g >= 0; g--) {
        const long long i = base + g * stride;
        const fe binv = fe_montmul(inv, pre[g]);
        inv = fe_montmul(inv, bm[g]);
        if (i < n) emit(i, binv);
    }
}

// ---- multi-point evaluation over the same tree (fast_evaluate, ntt.py:82-100, and M'(d_i) of fast_interpolate) ----
// The reference walks DOWN a remainder tree (f mod left zerofier, f mod right zerofier, ...).  Here the walk down is
// the TRANSPOSE of the interpolation up-sweep (Bostan-Lecerf-Schost): the up-sweep q -> P = sum q_i M / (X - d_i) is
// linear, rev(P) / rev(M) = sum q_i / (1 - d_i x) has the power sums sum_i q_i d_i^j as coefficients, i.e.
// (transposed Vandermonde) = (multiply by alpha = 1 / rev(M) mod x^n) o (reverse) o (up-sweep), so
//   f(d_i) = (up-sweep)^T [ (rev(f) * alpha mod x^n) shifted ],
// and the transposed up-sweep turns every product P_L * M_R into a CORRELATION with M_R: with the node transforms
// kept from the build, c_L = IDFT(DFT(c_node)[t] * DFT(M_R)[-t])[0..m) (+ c_node[m..2m) for the implied leading 1 of
// a full M_R), c_R likewise with M_L.  No division anywhere: one power-series inverse (Newton) at the top, then per
// level one batched forward transform, one pointwise kernel, one batched inverse transform, one fix-up.
// W (two blocks of 4s): [0] = rev_k(z) mod x^2s, zero padded; [1] = alpha mod x^s, zero padded.  z has k + 1
// coefficients.  (idx < 8s)
SA_HD void series_pad_elem(fe *W, const fe *z, long long k, const fe *alpha, long long s, long long idx) {
    const long long n4 = 4 * s, t = idx & (n4 - 1);
    fe v = fe_zero();
    if (idx < n4) {
        if (t < 2 * s && t <= k) v = tile_ld(z + (k - t));
    } else if (t < s) {
        v = tile_ld(alpha + t);
    }
    tile_st(W + idx, v);
}
// Newton step in the transform domain: W[0][t] = a * (2 - r * a), r = W[0][t], a = W[1][t]  (degree < 4s: no wrap)
SA_HD void series_step_elem(fe *W, long long n4, long long t) {
    const fe two = fe_make(2, 0, 0, 0);
    const fe r = tile_ld(W + t), a_m = fe_to_mont(tile_ld(W + n4 + t));
    const fe ra = fe_montmul(a_m, r);  // canonical r * a
    tile_st(W + t, fe_montmul(a_m, fe_sub(two, ra)));
}
// W (two blocks of n2): [0] = rev_{n-1}(f) (f has nf <= n coefficients), [1] = alpha mod x^n, both zero padded
SA_HD void eval_top_pad_elem(fe *W, const fe *f, long long nf, const fe *alpha, long long n, long long n2,
                             long long idx) {
    const long long t = idx & (n2 - 1);
    fe v = fe_zero();
    if (idx < n2) {
        if (t < n && n - 1 - t < nf) v = tile_ld(f + (n - 1 - t));
    } else if (t < n) {
        v = tile_ld(alpha + t);
    }
    tile_st(W + idx, v);
}
// root vector of the walk down: c[i] = s[n - k + i] for i < k (s = rev(f) * alpha), 0 for the empty slots
SA_HD void eval_root_elem(fe *c, const fe *s, long long n, long long k, long long i) {
    tile_st(c + i, i < k ? tile_ld(s + (n - k + i)) : fe_zero());
}
// O[child][t] = chat[parent][t] * VT[sibling][(2m - t) mod 2m]   (child blocks of 2m; VT = level-mlog transforms)
SA_HD void tree_down_elem(fe *O, const fe *chat, const fe *VT, int mlog, long long idx) {
    const long long two_m = 2ll << mlog, child = idx >> (mlog + 1), t = idx & (two_m - 1);
    const fe a = tile_ld(chat + (child >> 1) * two_m + t);
    const fe b = tile_ld(VT + (child ^ 1) * two_m + ((two_m - t) & (two_m - 1)));
    tile_st(O + idx, fe_montmul(fe_to_mont(a), b));
}
// next[child][j] = O[child][j] + [sibling full] * cur[parent][m + j],  j < m  (idx < K)
SA_HD void tree_down_fix_elem(fe *next, const fe *O, const fe *cur, int mlog, long long k, long long idx) {
    const long long m = 1ll << mlog, child = idx >> mlog, j = idx & (m - 1);
    fe v = tile_ld(O + child * 2 * m + j);
    if (tree_full(child ^ 1, mlog, k)) v = fe_add(v, tile_ld(cur + (child >> 1) * 2 * m + m + j));
    tile_st(next + idx, v);
}

// ---- host schedule ----
constexpr int TREE_MAX_LOG = 20;  // 2^20 points: ~1 GiB of tree, transforms and scratch

// primitive 2^log-th root of unity: generator^(2^119 / 2^log), algebra.py:100-114
inline const uint64_t *tree_root_of_unity(int log) {
    // algebra.py:100-102: generator 85408008396924667383611388730472331217 has order 2^119; the table is built
    // once (a tree of 2^16 points asks ~60 times per call, each a chain of up to 118 host-side squarings)
    static uint64_t table[120][2];
    static std::once_flag once;
    std::call_once(once, [] {
        const uint64_t g[2] = {0xb5038f9c18f6f7d1ull, 0x4040fbed12ee470full};
        fe w = fe_to_mont(fe_from_limbs(g));
        for (int i = 119; i >= 0; i--) {
            const fe c = fe_from_mont(w);
            table[i][0] = (uint64_t)c.v[0] | ((uint64_t)c.v[1] << 32);
            table[i][1] = (uint64_t)c.v[2] | ((uint64_t)c.v[3] << 32);
            w = fe_montmul(w, w);
        }
    });
    return table[log];
}

inline size_t sec16(size_t elems) { return (elems + 15) & ~(size_t)15; }  // rounded to 256 bytes

// The tree of one call over k points and its workspace ws (element offsets into it):
//   levels ((log K + 1) * K: level j at + j * K, the root at level log K)
//   | node transforms, on a 256-byte boundary: every level's (log K * 2K, level j at + j * 2K) where the walk reads
//     them (TREE_EVAL), one level's at a time (2K, TREE_ZEROFIER), none where they go into a plan (TREE_PLAN)
//   | z = the root's k + 1 coefficients (K + 1), for a plan dz = z' and ev = z'(d_i) (K each)
//   | the walk's W (4N), alpha (N), c0, c1 (K each), N = 2^ceil(log2 max(nf, k)); nf = 0: no walk.
// z, and the walk of TREE_EVAL, start on 256-byte boundaries; a plan packs z, dz, ev and the walk back to back.
// elems = 0: more than 2^TREE_MAX_LOG points.
enum TreeJob { TREE_ZEROFIER, TREE_PLAN, TREE_EVAL };
struct Tree {
    TreeJob job;
    int logK;
    long long k, K;
    size_t transforms, z, dz, ev, walk, elems;
    fe *ws, *plan;  // the workspace (elems elements); a plan's node transforms (TREE_PLAN)
    fe *level(int j) const { return ws + (size_t)j * K; }
    fe *node_transforms(int j) const {
        const size_t at = (size_t)j * 2 * K;
        return job == TREE_PLAN ? plan + at : ws + transforms + (job == TREE_EVAL ? at : 0);
    }
};
inline Tree tree_layout(size_t k, TreeJob job, size_t nf) {
    Tree t{job, host_log2(k), (long long)k, 0, 0, 0, 0, 0, 0, 0, nullptr, nullptr};
    t.K = 1ll << t.logK;
    if (t.logK > TREE_MAX_LOG) return t;
    const size_t K = (size_t)t.K, logK = (size_t)t.logK;
    t.transforms = sec16((logK + 1) * K);
    t.z = t.transforms + sec16(job == TREE_EVAL ? logK * 2 * K : job == TREE_ZEROFIER ? 2 * K : 0);
    t.dz = t.z + K + 1;
    t.ev = t.dz + K;
    t.walk = job == TREE_PLAN ? t.ev + K : job == TREE_EVAL ? t.z + sec16(K + 1) : t.z;
    t.elems = t.walk + (nf ? 5 * ((size_t)1 << host_log2(std::max(nf, k))) + 2 * K : 0);
    return t;
}

// builds every level of the zerofier tree of domain[0..k)
template <class B>
int tree_build(B &b, const Tree &t, const fe *domain) {
    const long long K = t.K;
    SA_TRY(b.leaves(t.level(0), domain, t.k, K));
    for (int j = 0; j < t.logK; j++) {
        const uint64_t *root = tree_root_of_unity(j + 1);
        fe *T = t.node_transforms(j), *child = t.level(j), *parent = t.level(j + 1);
        SA_TRY(b.pad(T, child, K, j));
        SA_TRY(b.ntt(T, T, j + 1, root, 0, (size_t)(K >> j)));
        SA_TRY(b.pairmul(parent, T, K, j));
        SA_TRY(b.ntt(parent, parent, j + 1, root, 1, (size_t)(K >> (j + 1))));
        SA_TRY(b.fix(parent, child, K, 1, j, t.k));
    }
    return SA_OK;
}

// vals[i] = f(d_i), i < k, for the tree `t` (built, its transforms kept) whose root polynomial is z (k + 1
// coefficients); f has nf >= 1 coefficients, and t was laid out with nf.  See the element functions' comment.
template <class B>
int tree_multipoint(B &b, const Tree &t, const fe *z, const fe *f, size_t nf, fe *vals) {
    const long long k = t.k, K = t.K;
    const long long n = (long long)std::max(nf, (size_t)k), N = 1ll << host_log2((size_t)n);
    fe *W = t.ws + t.walk, *alpha = W + 4 * N, *c0 = alpha + N, *c1 = c0 + K;
    // alpha = 1 / rev_k(z) mod x^N by Newton: alpha_2s = alpha_s (2 - r alpha_s) mod x^2s in transforms of size 4s
    SA_TRY(b.store(alpha, fe_one()));
    for (long long s = 1; s < N; s <<= 1) {
        const int lg = host_log2((size_t)(4 * s));
        const uint64_t *root = tree_root_of_unity(lg);
        SA_TRY(b.series_pad(W, z, k, alpha, s));
        SA_TRY(b.ntt(W, W, lg, root, 0, 2));
        SA_TRY(b.series_step(W, 4 * s));
        SA_TRY(b.ntt(W, W, lg, root, 1, 1));
        SA_TRY(b.copy(alpha, W, (size_t)(2 * s)));
    }
    // s = rev_{n-1}(f) * alpha mod x^n; the walk starts from c_root[i] = s[n - k + i]
    const long long n2 = 2 * N;
    const int lg = host_log2((size_t)n2);
    const uint64_t *root = tree_root_of_unity(lg);
    SA_TRY(b.eval_top_pad(W, f, (long long)nf, alpha, n, n2));
    SA_TRY(b.ntt(W, W, lg, root, 0, 2));
    SA_TRY(b.pointwise_mul(W, W, W + n2, n2));
    SA_TRY(b.ntt(W, W, lg, root, 1, 1));
    SA_TRY(b.eval_root(c0, W, n, k, K));
    // walk down: level j + 1 (nodes of 2m) -> level j (nodes of m); W is free again: chat = W[0, K), O = W[K, 3K)
    fe *cur = c0, *nxt = c1, *chat = W, *O = W + K;
    for (int j = t.logK - 1; j >= 0; j--) {
        const uint64_t *rootj = tree_root_of_unity(j + 1);
        SA_TRY(b.ntt(chat, cur, j + 1, rootj, 0, (size_t)(K >> (j + 1))));
        SA_TRY(b.down(O, chat, t.node_transforms(j), K, j));
        SA_TRY(b.ntt(O, O, j + 1, rootj, 1, (size_t)(K >> j)));
        SA_TRY(b.down_fix(nxt, O, cur, K, j, k));
        std::swap(cur, nxt);
    }
    return b.copy(vals, cur, (size_t)k);
}

// prod (X - d_i) (k + 1 coefficients) by the tree t (TREE_ZEROFIER)
template <class B>
int tree_zerofier(B &b, const Tree &t, fe *out, const fe *domain) {
    SA_TRY(tree_build(b, t, domain));
    return b.root(out, t.level(t.logK), t.k, t.K);
}

// f(points[i]) by the walk down the tree t (TREE_EVAL, laid out with nf); f has nf >= 1 coefficients
template <class B>
int tree_poly_eval(B &b, const Tree &t, fe *out, const fe *f, size_t nf, const fe *points) {
    SA_TRY(tree_build(b, t, points));
    SA_TRY(b.root(t.ws + t.z, t.level(t.logK), t.k, t.K));
    return tree_multipoint(b, t, t.ws + t.z, f, nf, out);
}

// ---- interpolation plans: the half of fast_interpolate (ntt.py:102-130) that depends on the domain alone ----
// A plan is a device buffer of sa_interp_plan_bytes(k) bytes, laid out by k alone.  Every section starts on a
// 256-byte (16-element) boundary, i.e. each section's length is rounded up to a multiple of 16 elements:
//   k <= INTERP_DIRECT_MAX (the k x k Lagrange kernels):  domain (k) | z = prod (X - d_i) (k + 1) | 1/z'(d_i) (k)
//   above (the subproduct tree):  node transforms of levels 0 .. log K - 1, as tree_build keeps them (log K * 2K)
//                                 | 1/M'(d_i) (K; the first k are written)
// The inverses are in Montgomery form, so one product per point gives v_i / M'(d_i).  The tree's levels and z stay
// in the build's workspace: the up-sweep reads the node transforms only.  2^20 points: 41 * 2^20 elements, 656 MiB.
constexpr size_t INTERP_DIRECT_MAX = 1024;
struct InterpPlan {
    bool direct = false;
    int logK = 0;
    long long K = 0;
    size_t sec[3] = {0, 0, 0};  // element offsets: domain, z, 1/z'  |  transforms, 1/M'
    size_t elems = 0;           // 0: no plan for this k
};
// force_tree: the tree's layout at any k >= 1 (the emulation runs trees of a few points)
inline InterpPlan interp_plan_layout(size_t k, bool force_tree = false) {
    InterpPlan L;
    if (k == 0 || k > ((size_t)1 << TREE_MAX_LOG)) return L;
    L.direct = k <= INTERP_DIRECT_MAX && !force_tree;
    if (L.direct) {
        L.sec[1] = sec16(k);
        L.sec[2] = L.sec[1] + sec16(k + 1);
        L.elems = L.sec[2] + sec16(k);
    } else {
        L.logK = host_log2(k);
        L.K = 1ll << L.logK;
        L.sec[1] = sec16((size_t)L.logK * 2 * (size_t)L.K);
        L.elems = L.sec[1] + sec16((size_t)L.K);
    }
    return L;
}

// M = prod (X - d_i) by the tree t (TREE_PLAN; its node transforms go into the plan), M'(d_i) by Horner (k^2 / 2
// multiply-adds, all points in parallel) or the walk down the tree (t laid out with nf = k), then one batch
// inversion; coinciding points give M'(d_i) = 0 -> *flag (SA_EDIVZERO like the division at ntt.py:124-125)
template <class B>
int interp_plan_tree(B &b, Tree t, fe *plan, const InterpPlan &L, const fe *domain, bool walk, int *flag) {
    t.plan = plan + L.sec[0];
    const long long k = t.k;
    fe *z = t.ws + t.z, *dz = t.ws + t.dz, *ev = t.ws + t.ev;
    SA_TRY(tree_build(b, t, domain));
    SA_TRY(b.root(z, t.level(t.logK), k, t.K));
    SA_TRY(b.derivative(dz, z, k));
    SA_TRY(walk ? tree_multipoint(b, t, z, dz, (size_t)k, ev) : b.horner(ev, dz, k, domain, k));
    return b.batch_inverse(plan + L.sec[1], ev, k, flag);
}

// Above the Lagrange kernels a batched apply needs 4K elements of its own workspace and 2K of the NTT's inter-pass
// intermediate per vector: 96K bytes.  It runs in chunks that keep both at or below 1 GiB.
constexpr size_t INTERP_CHUNK_BYTES = (size_t)1 << 30;
inline size_t interp_batch_max(const InterpPlan &L) {
    if (L.elems == 0) return 0;
    if (L.direct) return SIZE_MAX;
    const size_t b = INTERP_CHUNK_BYTES / (sizeof(fe) * 6 * (size_t)L.K);
    return b ? b : 1;
}
// the interpolants sum_i q_i M / (X - d_i), q_i = v_i / M'(d_i), of nb value vectors, combined bottom-up over the
// plan's tree: P_node = P_L * M_R + P_R * M_L.  Every level is one batch over the nodes of all nb trees, so the
// launches do not depend on nb.  ws = 4K * nb elements: transform scratch [nb][2K], P ping-pong 2 x [nb][K].
template <class B>
int interp_sweep(B &b, fe *out, const fe *p, const InterpPlan &L, const fe *v, size_t k, size_t nb, fe *ws) {
    const size_t K = (size_t)L.K;
    const long long n = (long long)(nb * K);
    fe *scratch = ws, *cur = ws + 2 * K * nb, *nxt = cur + K * nb;
    SA_TRY(b.qleaves(cur, v, p + L.sec[1], (long long)k, L.logK, (long long)nb));
    for (int j = 0; j < L.logK; j++) {
        const uint64_t *root = tree_root_of_unity(j + 1);
        SA_TRY(b.pad(scratch, cur, n, j));
        SA_TRY(b.ntt(scratch, scratch, j + 1, root, 0, nb * (K >> j)));
        SA_TRY(b.cross(nxt, scratch, p + L.sec[0] + (size_t)j * 2 * K, L.K, (long long)nb, j));
        SA_TRY(b.ntt(nxt, nxt, j + 1, root, 1, nb * (K >> (j + 1))));
        SA_TRY(b.fix(nxt, cur, L.K, (long long)nb, j, (long long)k));
        std::swap(cur, nxt);
    }
    return b.copy2d(out, k, cur, K, k, nb);
}
// `batch` vectors through the tree of a plan, in chunks of interp_batch_max(L); ws = 4K per vector of a chunk
template <class B>
int interp_apply_tree(B &b, fe *out, const fe *p, const InterpPlan &L, const fe *v, size_t k, size_t batch, fe *ws) {
    const size_t chunk = std::min(batch, interp_batch_max(L));
    for (size_t b0 = 0; b0 < batch; b0 += chunk)
        SA_TRY(interp_sweep(b, out + b0 * k, p, L, v + b0 * k, k, std::min(chunk, batch - b0), ws));
    return SA_OK;
}

}  // namespace sa
