// geo.cuh -- interpolation over, and the zerofier of, a geometric domain 1, q, q^2, ..., q^(k-1): the per-element
// bodies of their kernels, a prefix-product scan over the field, and the host schedules of the plan build, the
// batched apply and the zerofier.  The library (poly.cu) runs the schedules with kernel launches, the CPU emulation
// (tests/emu) with loops over the element functions.
//
// The schedules take the backend of poly_tree.cuh and coset.cuh (one method per kernel, named after it without the
// k_ prefix: k_geo_load -> b.geo_load; k_pow_table -> b.pow_table(out, base_m, count); k_batch_inverse ->
// b.batch_inverse; k_coset_quot -> b.coset_quot; b.ntt as sa_ntt; b.copy2d).
//
// With (q;q)_m = prod_{d=1..m} (1 - q^d) and C(t) = t (t - 1) / 2 (the q-binomial theorem):
//   Z(x) = prod_{i<k} (x - q^i) has z_{k-j} = (-1)^j q^C(j) (q;q)_k / ((q;q)_j (q;q)_{k-j}),  0 <= j <= k;
//   c_i = (-1)^i (q^(2-k))^i / ((q;q)_i (q;q)_{k-1-i}) = q^-C(i) / Z'(q^i);
// and the interpolant f of values v (degree < k) is, with u_i = v_i c_i,
//   m_j = q^-C(j) sum_i u_i q^C(i+j)      (j < k; ij = C(i+j) - C(i) - C(j), so m_j = sum_i (v_i / Z'(q^i)) q^ij)
//   f_j = sum_{t<k-j} z_{j+1+t} m_t       (j < k; the polynomial part of Z(x) sum_t m_t x^(-t-1))
// -- two middle products, each one cyclic convolution of length K = 2^ceil(log2 2k): reversed u against the chirp
// q^C(t), t < 2k - 1, read at k - 1 + j (the wrapped tail of the product ends below k - 1 since K >= 2k - 1), then
// reversed m against z, read at k + j (the product has 2k coefficients: no wrap).  f is the unique interpolant, so
// its coefficients are those of the subproduct tree's apply, bit for bit.
//
// The method needs q^d != 1 for 1 <= d <= k (else some (q;q)_m = 0) and q != 0 from k = 2 on.  q^d != 1 for d < k
// is exactly "the k points are distinct"; d = k is one more: a step of order exactly k spans a whole subgroup, whose
// interpolation is an inverse NTT, and is refused here although the tree interpolates it.
#pragma once
#include <algorithm>
#include <cstdint>

#include "coset.cuh"
#include "host.cuh"
#include "ntt_tile.cuh"
#include "poly_tree.cuh"

namespace sa {

// ---- the prefix-product scan: x[i] <- x[0] * ... * x[i] (Montgomery form in, Montgomery form out) ----
// Level l holds n_l elements in runs of GEO_SCAN_RUN; a thread scans one run in place and writes its product to level
// l + 1 (n_{l+1} = ceil(n_l / RUN)), down to a single element; then, from the top down, every element of run r >= 1
// of level l is multiplied by the scanned element r - 1 of level l + 1.
constexpr int GEO_SCAN_RUN = 16;
// run r of x[0..n) scanned in place, its product into tot[r]  (r < ceil(n / RUN))
SA_HD void geo_scan_run_elem(fe *x, long long n, fe *tot, long long r) {
    const long long i0 = r * GEO_SCAN_RUN;
    fe acc = tile_ld(x + i0);
    for (long long i = i0 + 1; i < i0 + GEO_SCAN_RUN && i < n; i++) {
        acc = fe_montmul(acc, tile_ld(x + i));
        tile_st(x + i, acc);
    }
    tile_st(tot + r, acc);
}
// x[i] *= tot[i / RUN - 1] for i = RUN + idx: the product of every run before i's  (idx < n - RUN)
SA_HD void geo_scan_add_elem(fe *x, const fe *tot, long long idx) {
    const long long i = idx + GEO_SCAN_RUN;
    tile_st(x + i, fe_montmul(tile_ld(x + i), tile_ld(tot + i / GEO_SCAN_RUN - 1)));
}

// ---- element functions of the plan build (everything in Montgomery form but the inverses, see geo_plan_build) ----
// P[m] = 1 - q^m for 1 <= m, P[0] = 1 (pw_m = q^m)  (m < count)
SA_HD void geo_factor_elem(fe *P, const fe *pw_m, long long m) {
    tile_st(P + m, m == 0 ? fe_mont_one() : fe_sub(fe_mont_one(), tile_ld(pw_m + m)));
}
// out[t] = 1 for t = 0, pw_m[t - 1] for 1 <= t < n, 0 up to len: scanned, q^C(t) (pw_m = q^t) or q^-C(t) (q^-t)
// (t < len)
SA_HD void geo_seed_elem(fe *out, const fe *pw_m, long long n, long long t) {
    tile_st(out + t, t == 0 ? fe_mont_one() : t < n ? tile_ld(pw_m + t - 1) : fe_zero());
}
// x_m / (a b) in Montgomery form, ia = 1/a and ib = 1/b canonical (batch_inverse of Montgomery-form a and b)
SA_HD fe geo_div2(const fe &x_m, const fe &ia, const fe &ib) {
    return fe_montmul(fe_montmul(x_m, fe_to_mont(ia)), fe_to_mont(ib));
}
// z[i] = the coefficient of x^i of prod_{d<k} (x - q^d) for i <= k, 0 from k + 1 up to len (a spectrum's padding):
// j = k - i; 1 for j = 0, (-1)^k q^C(k) for j = k, else (-1)^j q^C(j) P_k / (P_j P_{k-j}) with P_m = (q;q)_m; chirp_m
// = q^C(t) for t <= k, P_m = (q;q)_m for m <= k, iP = 1/(q;q)_m canonical for m < k.  Montgomery form, or canonical
// with canon != 0  (i < len)
SA_HD void geo_zerofier_elem(fe *z, const fe *chirp_m, const fe *P_m, const fe *iP, long long k, int canon,
                             long long i) {
    fe v = fe_zero();
    if (i <= k) {
        const long long j = k - i;
        if (j == 0) {
            v = fe_mont_one();
        } else {
            v = j == k ? tile_ld(chirp_m + k)
                       : geo_div2(fe_montmul(tile_ld(chirp_m + j), tile_ld(P_m + k)), tile_ld(iP + j), tile_ld(iP + i));
            if (j & 1) v = fe_neg(v);
        }
        if (canon) v = fe_from_mont(v);
    }
    tile_st(z + i, v);
}
// c[i] = (-1)^i E_i / (P_i P_{k-1-i}) in place, E_i = (q^(2-k))^i (Montgomery form; the buffer holds E on entry),
// iP = 1/(q;q)_m canonical  (i < k)
SA_HD void geo_weight_elem(fe *c, const fe *iP, long long k, long long i) {
    const fe v = geo_div2(tile_ld(c + i), tile_ld(iP + i), tile_ld(iP + (k - 1 - i)));
    tile_st(c + i, (i & 1) ? fe_neg(v) : v);
}

// ---- element functions of the apply, over rows of K = 2^logK ----
// ws[b][i] = v_b[k-1-i] c[k-1-i] for i < k, 0 up to K: u reversed and padded (values canonical, c_m Montgomery)
// (idx < batch * K)
SA_HD void geo_load_elem(fe *ws, const fe *values, const fe *c_m, long long k, int logK, long long idx) {
    const long long b = idx >> logK, i = idx & ((1ll << logK) - 1);
    tile_st(ws + idx,
            i < k ? fe_montmul(tile_ld(values + b * k + (k - 1 - i)), tile_ld(c_m + (k - 1 - i))) : fe_zero());
}
// dst[b][i] = m_b[k-1-i] for i < k, 0 up to K: m_j = q^-C(j) y[k-1+j] (ic_m = q^-C(j), y = src, the first product)
// extracted, reversed and padded  (idx < batch * K)
SA_HD void geo_mid_elem(fe *dst, const fe *src, const fe *ic_m, long long k, int logK, long long idx) {
    const long long b = idx >> logK, i = idx & ((1ll << logK) - 1);
    tile_st(dst + idx, i < k ? fe_montmul(tile_ld(src + (b << logK) + (2 * k - 2 - i)), tile_ld(ic_m + (k - 1 - i)))
                             : fe_zero());
}

// ---- host schedule ----
// 2^26 points: K = 2^27, a plan of 6 GiB and an apply of 6 GiB per vector.
constexpr int GEO_MAX_LOG = 26;

// A plan is a device buffer of geo_plan_layout(k).elems elements, laid out by k alone; every section starts on a
// 256-byte (16-element) boundary:  c (k) | q^-C(j) (k) | DFT_K(q^C(t), t < 2k - 1) (K) | DFT_K(z) (K), all in
// Montgomery form, so each product of an apply is one fe_montmul.  16 (2k + 2K) bytes up to the rounding: 96 MiB at
// k = 2^20.
struct GeoPlan {
    int logK = 0;
    long long k = 0, K = 0;
    size_t c = 0, ic = 0, chirp = 0, zs = 0;  // element offsets of the sections
    size_t elems = 0;                          // 0: no plan for this k
};
inline GeoPlan geo_plan_layout(size_t k) {
    GeoPlan L;
    if (k == 0 || k > ((size_t)1 << GEO_MAX_LOG)) return L;
    L.k = (long long)k;
    L.logK = host_log2(2 * k);
    L.K = 1ll << L.logK;
    L.ic = sec16(k);
    L.chirp = 2 * L.ic;
    L.zs = L.chirp + (size_t)L.K;
    L.elems = L.zs + (size_t)L.K;
    return L;
}

// A chunk of an apply takes 2K elements of its own workspace and K of the NTT's inter-pass intermediate per vector:
// 48 K bytes.  It runs in chunks that keep both at or below 1 GiB.
constexpr size_t GEO_CHUNK_BYTES = (size_t)1 << 30;
inline size_t geo_batch_max(size_t k) {
    const GeoPlan L = geo_plan_layout(k);
    if (L.elems == 0) return 0;
    const size_t b = GEO_CHUNK_BYTES / (sizeof(fe) * 3 * (size_t)L.K);
    return b ? b : 1;
}

// The checks of a plan build or a zerofier, before any workspace is taken and before the first launch: k in
// 1..2^26 (SA_ESIZE), step != 0 from k = 2 on (SA_EDIVZERO: the points 1, 0, 0, ... coincide).
inline int geo_check(size_t k, const uint64_t step[2]) {
    if (k == 0 || k > ((size_t)1 << GEO_MAX_LOG)) return SA_ESIZE;
    return k >= 2 && fe_is_zero(fe_to_mont(fe_from_limbs(step))) ? SA_EDIVZERO : SA_OK;
}

// the scan's levels above x: ceil(n / RUN) + ceil(ceil(n / RUN) / RUN) + ... down to one element
inline size_t geo_scan_elems(long long n) {
    size_t e = 0;
    while (n > 1) {
        n = (n + GEO_SCAN_RUN - 1) / GEO_SCAN_RUN;
        e += (size_t)n;
    }
    return e;
}
// x[0..n) <- its prefix products (Montgomery form); tmp = geo_scan_elems(n) elements.  2 launches per level.
template <class B>
int geo_scan(B &b, fe *x, long long n, fe *tmp) {
    constexpr int MAXL = 64;
    fe *lv[MAXL];
    long long ln[MAXL];
    int L = 0;
    lv[0] = x;
    ln[0] = n;
    fe *next = tmp;
    while (ln[L] > 1) {
        ln[L + 1] = (ln[L] + GEO_SCAN_RUN - 1) / GEO_SCAN_RUN;
        lv[L + 1] = next;
        next += ln[L + 1];
        SA_TRY(b.geo_scan_runs(lv[L], ln[L], lv[L + 1]));
        L++;
    }
    for (int l = L - 2; l >= 0; l--) SA_TRY(b.geo_scan_add(lv[l], ln[l], lv[l + 1]));
    return SA_OK;
}

// The build's workspace: q^t (max(k + 1, nc) with nc the chirp's length), (q;q)_m and its inverses (k + 1 each) and
// the scan's levels (of the longest scan, nc elements).
struct GeoWork {
    long long nc = 0;
    size_t pw = 0, P = 0, iP = 0, scan = 0, elems = 0;
};
inline GeoWork geo_work_layout(size_t k, long long nc) {
    GeoWork w;
    w.nc = nc;
    w.P = sec16(std::max((size_t)nc, k + 1));
    w.iP = w.P + sec16(k + 1);
    w.scan = w.iP + sec16(k + 1);
    w.elems = w.scan + geo_scan_elems(nc);
    return w;
}
// the chirp's length: q^C(t) for t < 2k - 1 (the first product) and t <= k (the zerofier's q^C(k))
inline long long geo_chirp_len(size_t k, bool plan) {
    return plan ? std::max(2 * (long long)k - 1, (long long)k + 1) : (long long)k + 1;
}

// what the plan and the zerofier share: q^t for t < max(k + 1, nc) into ws.pw, (q;q)_m for m <= k into ws.P (one
// scan), their inverses (canonical: the batch inversion of Montgomery-form values) into ws.iP -- a zero (q;q)_m, i.e.
// q^d = 1 for some d <= m, raises *flag; m < k only for k = 1, whose one point is never refused -- and the chirp
// q^C(t), t < nc, scanned in chirp (nc elements, zero up to len).
template <class B>
int geo_common(B &b, const GeoWork &w, fe *ws, const fe &q_m, size_t k, fe *chirp, long long len, int *flag) {
    fe *pw = ws + w.pw, *P = ws + w.P, *iP = ws + w.iP, *tmp = ws + w.scan;
    SA_TRY(b.pow_table(pw, q_m, std::max((long long)k + 1, w.nc)));
    SA_TRY(b.geo_factor(P, pw, (long long)k + 1));
    SA_TRY(geo_scan(b, P, (long long)k + 1, tmp));
    SA_TRY(b.batch_inverse(iP, P, k >= 2 ? (long long)k + 1 : (long long)k, flag));
    SA_TRY(b.geo_seed(chirp, pw, w.nc, len));
    return geo_scan(b, chirp, w.nc, tmp);
}

// The plan of (step, k) into plan (geo_plan_layout(k).elems elements), ws = geo_work_layout(k, geo_chirp_len(k,
// true)).elems elements; *flag as geo_common.  The plan's own sections serve as scratch on the way: the chirp is
// scanned where its transform goes, q^-t and (q^(2-k))^i go where c goes.
template <class B>
int geo_plan_build(B &b, fe *plan, const uint64_t step[2], size_t k, fe *ws, int *flag) {
    const GeoPlan L = geo_plan_layout(k);
    const GeoWork w = geo_work_layout(k, geo_chirp_len(k, true));
    const uint64_t *root = tree_root_of_unity(L.logK);
    const fe q_m = fe_to_mont(fe_from_limbs(step)), qi_m = fe_mont_inv(q_m);
    fe *c = plan + L.c, *ic = plan + L.ic, *chirp = plan + L.chirp, *zs = plan + L.zs;
    SA_TRY(geo_common(b, w, ws, q_m, k, chirp, L.K, flag));
    SA_TRY(b.geo_zerofier(zs, chirp, ws + w.P, ws + w.iP, L.k, 0, L.K));
    SA_TRY(b.pow_table(c, qi_m, L.k));
    SA_TRY(b.geo_seed(ic, c, L.k, L.k));
    SA_TRY(geo_scan(b, ic, L.k, ws + w.scan));
    SA_TRY(b.pow_table(c, fe_montmul(fe_montmul(q_m, q_m), fe_mont_pow_u64(qi_m, (uint64_t)k)), L.k));
    SA_TRY(b.geo_weight(c, ws + w.iP, L.k));
    // the chirp's tail beyond 2k - 1 (q^C(k) for k = 1) is read by no output: (k - 1 + j) - t >= 0 for t <= k - 1 + j
    SA_TRY(b.ntt(chirp, chirp, L.logK, root, 0, 1));
    return b.ntt(zs, zs, L.logK, root, 0, 1);
}

// the k + 1 coefficients of prod_{i<k} (x - step^i) into out (canonical), ws = geo_work_layout(k, geo_chirp_len(k,
// false)).elems + k + 1 elements (the chirp after the build's workspace).  The flag is read between the two halves
// (check(flag) returns SA_OK or the error), so an error leaves out untouched.
template <class B, class Check>
int geo_zerofier(B &b, fe *out, const uint64_t step[2], size_t k, fe *ws, int *flag, Check check) {
    const GeoWork w = geo_work_layout(k, geo_chirp_len(k, false));
    fe *chirp = ws + w.elems;
    SA_TRY(geo_common(b, w, ws, fe_to_mont(fe_from_limbs(step)), k, chirp, w.nc, flag));
    SA_TRY(check(flag));
    return b.geo_zerofier(out, chirp, ws + w.P, ws + w.iP, (long long)k, 1, (long long)k + 1);
}

// `batch` value vectors through a plan: out[b] = f_b (k coefficients each).  Per chunk of geo_batch_max(k) vectors:
// load, transform, product with the chirp's spectrum, inverse transform, extract, transform, product with z's
// spectrum, inverse transform, one strided copy -- the same launches whatever the chunk's size.  ws = 2K elements
// per vector of a chunk of `chunk` vectors (the library's: geo_batch_max(k)).
template <class B>
int geo_apply(B &b, fe *out, const fe *plan, const fe *values, size_t k, size_t batch, fe *ws, size_t chunk) {
    const GeoPlan L = geo_plan_layout(k);
    const uint64_t *root = tree_root_of_unity(L.logK);
    const size_t K = (size_t)L.K;
    chunk = std::min(batch, chunk);
    fe *A = ws, *Bv = ws + K * chunk;
    for (size_t b0 = 0; b0 < batch; b0 += chunk) {
        const size_t nb = std::min(chunk, batch - b0);
        SA_TRY(b.geo_load(A, values + b0 * k, plan + L.c, L.k, L.logK, (long long)nb));
        SA_TRY(b.ntt(A, A, L.logK, root, 0, nb));
        SA_TRY(b.coset_quot(A, plan + L.chirp, L.logK, (long long)nb));
        SA_TRY(b.ntt(A, A, L.logK, root, 1, nb));
        SA_TRY(b.geo_mid(Bv, A, plan + L.ic, L.k, L.logK, (long long)nb));
        SA_TRY(b.ntt(Bv, Bv, L.logK, root, 0, nb));
        SA_TRY(b.coset_quot(Bv, plan + L.zs, L.logK, (long long)nb));
        SA_TRY(b.ntt(Bv, Bv, L.logK, root, 1, nb));
        SA_TRY(b.copy2d(out + b0 * k, k, Bv + k, K, k, nb));
    }
    return SA_OK;
}

}  // namespace sa
