// coset.cuh -- division by one polynomial on a coset, many numerators at a time (fast_coset_divide,
// code/ntt.py:137-176), batched coset evaluation (fast_coset_evaluate, ntt.py:132-135) and the coset evaluation of a
// weighted, degree-shifted sum of many polynomials (fast_stark.py:125-148): the per-element bodies of their kernels
// and the host schedules of the plan build, the apply, the evaluation and the combination.  The library (poly.cu)
// runs the schedules with kernel launches, the CPU emulation (tests/emu) with loops over the element functions.
//
// The schedules take the backend of poly_tree.cuh (one method per kernel, named after it without the k_ prefix:
// k_coset_load -> b.coset_load; k_pow_table -> b.pow_table(out, base_m, count), lead 1, natural order;
// k_batch_inverse -> b.batch_inverse; b.ntt as sa_ntt).
//
// With n = 2^log_n, R_i = r(offset * root^i) and L_i = l(offset * root^i), row b of an apply is
//     out[b][j] = U[j] * offset^-j  (j < qlen),   U = intt(L_i / R_i),
// i.e. fast_coset_divide before its truncation, at order n.  Everything that depends on (r, offset, root, n) alone
// -- offset^i, 1/R_i, offset^-i -- is the plan; per numerator there remain two transforms and three streaming
// kernels, and no host synchronisation.
#pragma once
#include <algorithm>
#include <cstdint>

#include "host.cuh"
#include "ntt_plan.cuh"
#include "ntt_tile.cuh"

namespace sa {

// ---- element functions: the body of each kernel for one index ----
// ws[b][i] = lhs[b][i] * offset^i for i < ncoef, 0 up to n (pw_m = offset^i in Montgomery form)  (idx < batch * n)
SA_HD void coset_load_elem(fe *ws, const fe *lhs, const fe *pw_m, long long ncoef, int log_n, long long idx) {
    const long long b = idx >> log_n, i = idx & ((1ll << log_n) - 1);
    tile_st(ws + idx, i < ncoef ? fe_montmul(tile_ld(lhs + b * ncoef + i), tile_ld(pw_m + i)) : fe_zero());
}
// ws[b][i] *= 1/R_i (inv_m = the plan's 1/R_i in Montgomery form, broadcast over the rows)  (idx < batch * n)
SA_HD void coset_quot_elem(fe *ws, const fe *inv_m, int log_n, long long idx) {
    tile_st(ws + idx, fe_montmul(tile_ld(ws + idx), tile_ld(inv_m + (idx & ((1ll << log_n) - 1)))));
}
// out[b][j] = ws[b][j] * offset^-j for j < qlen (ipw_m = offset^-j in Montgomery form)  (idx < batch * n)
SA_HD void coset_store_elem(fe *out, const fe *ws, const fe *ipw_m, long long qlen, int log_n, long long idx) {
    const long long b = idx >> log_n, j = idx & ((1ll << log_n) - 1);
    if (j < qlen) tile_st(out + b * qlen + j, fe_montmul(tile_ld(ws + idx), tile_ld(ipw_m + j)));
}

// A group of a combination's terms, taken by one launch as a kernel parameter (__grid_constant__: 3 KB, inside the
// classic 4 KB parameter limit).  Term t is the row src[0..len) shifted up by `shift`, weighted by w_m (Montgomery
// form, so each covered index costs one fe_montmul and one fe_add), and added into destination row `row`.
constexpr int COMBINE_TERMS = 64;
struct CombineTerm {
    const fe *src;
    long long len, shift, row;
    fe w_m;
};
struct CombineGroup {
    CombineTerm t[COMBINE_TERMS];
    int count;
};
// out[r][i] (+)= offset^i * sum_t w_t * src_t[i - shift_t] over the group's terms of row r whose window covers i, for
// i < ncomb (the longest row's length; a shorter row's sum is zero past its own); the first group (first != 0)
// writes every i < n of every row, zero from ncomb on, each later one adds its own scaled sum (scaling by offset^i is
// linear)  (idx = r * n + i < nrows * n)
SA_HD void coset_combine_elem(fe *out, const CombineGroup &g, const fe *pw_m, long long ncomb, int first, int log_n,
                              long long idx) {
    const long long r = idx >> log_n, i = idx & ((1ll << log_n) - 1);
    if (i >= ncomb) {
        if (first) tile_st(out + idx, fe_zero());
        return;
    }
    fe s = fe_zero();
    for (int t = 0; t < g.count; t++) {
        const long long j = i - g.t[t].shift;
        if (g.t[t].row == r && j >= 0 && j < g.t[t].len) s = fe_add(s, fe_montmul(tile_ld(g.t[t].src + j), g.t[t].w_m));
    }
    s = fe_montmul(s, tile_ld(pw_m + i));
    tile_st(out + idx, first ? s : fe_add(tile_ld(out + idx), s));
}
// one row: out[i] for i < n, every term in row 0
SA_HD void coset_combine_elem(fe *out, const CombineGroup &g, const fe *pw_m, long long ncomb, int first, long long i) {
    coset_combine_elem(out, g, pw_m, ncomb, first, 62, i);
}

// ---- host schedule ----
// The transforms' range.  A plan is 48 n bytes (6 GiB at 2^27, 48 GiB at 2^30), so with the operands and the
// workspaces the largest sizes do not fit on one 80 GB device.
constexpr int COSET_MAX_LOG = NTT_MAX_LOG_N;

// A plan is a device buffer of coset_div_plan_layout(log_n).elems elements, laid out by log_n alone; every section
// starts on a 256-byte (16-element) boundary:  offset^i (n) | 1/R_i (n) | offset^-i (n), all in Montgomery form, so
// each kernel of an apply does one fe_montmul per element and takes no scalar.  48 n bytes from n = 16 on.
struct CosetPlan {
    int log_n = 0;
    long long n = 0;
    size_t pw = 0, inv = 0, ipw = 0;  // element offsets of the sections
    size_t elems = 0;                 // 0: no plan for this log_n
};
inline CosetPlan coset_div_plan_layout(int log_n) {
    CosetPlan L;
    if (log_n < 1 || log_n > COSET_MAX_LOG) return L;
    L.log_n = log_n;
    L.n = 1ll << log_n;
    L.inv = sec16((size_t)L.n);
    L.ipw = 2 * L.inv;
    L.elems = 3 * L.inv;
    return L;
}

// A chunk of an apply or evaluation takes 16 bytes per element per row of its own workspace (the transformed rows;
// an evaluation transforms in `out` instead) and 16 of the NTT's inter-pass intermediate: 32 n bytes per row.  It
// runs in chunks that keep both at or below 1 GiB.
constexpr size_t COSET_CHUNK_BYTES = (size_t)1 << 30;
inline size_t coset_batch_max(int log_n) {
    if (log_n < 1 || log_n > COSET_MAX_LOG) return 0;
    const size_t b = COSET_CHUNK_BYTES / (2 * sizeof(fe) << log_n);
    return b ? b : 1;
}

// The checks of every call, made before its workspaces are taken and before its first launch: the size, the
// coefficient counts (1..n) and the root (sa_ntt's SA_EROOTORDER / SA_ENOTPRIM).  The schedules below assume them.
inline int coset_check(int log_n, size_t ncoef, size_t qlen, const uint64_t root[2]) {
    if (log_n < 1 || log_n > COSET_MAX_LOG) return SA_ESIZE;
    const size_t n = (size_t)1 << log_n;
    if (ncoef < 1 || ncoef > n || qlen < 1 || qlen > n) return SA_ESIZE;
    return ntt_check_root(fe_to_mont(fe_from_limbs(root)), log_n);
}
// a plan build's: a divisor of 1..n coefficients.  Every offset is accepted, 0 included (see coset_div_plan_build).
inline int coset_div_plan_check(int log_n, size_t dlen, const uint64_t root[2], const uint64_t * /*offset*/) {
    return coset_check(log_n, dlen, 1, root);
}

// the plan of divisor[0..dlen) on the coset offset * <root>: the two power tables, then R = ntt(r_i * offset^i)
// in ws (n elements) and its batch inversion into the plan.  Some R_i = 0 (the zero divisor among them) raises
// *flag: the reference's l / r raises "divide by zero" there (algebra.py:92).  Offset 0 is the reference's too:
// its powers are 1, 0, 0, ... (scale keeps the constant term) and its inverse is 0 (algebra.py:87-89).
template <class B>
int coset_div_plan_build(B &b, fe *plan, const fe *divisor, size_t dlen, int log_n, const uint64_t root[2],
                         const uint64_t offset[2], fe *ws, int *flag) {
    const CosetPlan L = coset_div_plan_layout(log_n);
    const fe off_m = fe_to_mont(fe_from_limbs(offset));
    SA_TRY(b.pow_table(plan + L.pw, off_m, L.n));
    SA_TRY(b.pow_table(plan + L.ipw, fe_mont_inv(off_m), L.n));
    SA_TRY(b.coset_load(ws, divisor, plan + L.pw, (long long)dlen, log_n, 1));
    SA_TRY(b.ntt(ws, ws, log_n, root, 0, 1));
    return b.batch_inverse(plan + L.inv, ws, L.n, flag);
}

// `batch` numerators lhs[batch][ncoef] through a plan of (log_n, root): out[batch][qlen].  Per chunk of
// coset_batch_max(log_n) rows: load, one forward transform of the chunk, quotient, one inverse transform, store --
// the same five launches (plus the transforms' passes) whatever the chunk's size.  ws = n elements per row of a chunk.
template <class B>
int coset_div_apply(B &b, fe *out, const fe *plan, const fe *lhs, size_t ncoef, size_t qlen, int log_n,
                    const uint64_t root[2], size_t batch, fe *ws) {
    const CosetPlan L = coset_div_plan_layout(log_n);
    const size_t chunk = std::min(batch, coset_batch_max(log_n));
    for (size_t b0 = 0; b0 < batch; b0 += chunk) {
        const size_t nb = std::min(chunk, batch - b0);
        SA_TRY(b.coset_load(ws, lhs + b0 * ncoef, plan + L.pw, (long long)ncoef, log_n, (long long)nb));
        SA_TRY(b.ntt(ws, ws, log_n, root, 0, nb));
        SA_TRY(b.coset_quot(ws, plan + L.inv, log_n, (long long)nb));
        SA_TRY(b.ntt(ws, ws, log_n, root, 1, nb));
        SA_TRY(b.coset_store(out + b0 * qlen, ws, plan + L.ipw, (long long)qlen, log_n, (long long)nb));
    }
    return SA_OK;
}

// out[b] = ntt(coeffs[b][i] * offset^i, zero padded to n) for b < batch (fast_coset_evaluate at order n): offset^i
// for i < ncoef into pw (ncoef elements), then per chunk the apply's load straight into out and one transform in place
template <class B>
int coset_evaluate(B &b, fe *out, const fe *coeffs, size_t ncoef, int log_n, const uint64_t root[2],
                   const uint64_t offset[2], size_t batch, fe *pw) {
    if (batch == 0) return SA_OK;
    const size_t n = (size_t)1 << log_n, chunk = std::min(batch, coset_batch_max(log_n));
    SA_TRY(b.pow_table(pw, fe_to_mont(fe_from_limbs(offset)), (long long)ncoef));
    for (size_t b0 = 0; b0 < batch; b0 += chunk) {
        const size_t nb = std::min(chunk, batch - b0);
        SA_TRY(b.coset_load(out + b0 * n, coeffs + b0 * ncoef, pw, (long long)ncoef, log_n, (long long)nb));
        SA_TRY(b.ntt(out + b0 * n, out + b0 * n, log_n, root, 0, nb));
    }
    return SA_OK;
}

// ---- coset combinations (the combination of fast_stark.py:125-148 and its fast_coset_evaluate) ----
// ncomb = max_t(shifts[t] + lens[t]): the combination's length, and the offset^i its schedule tables
inline size_t coset_combine_len(const size_t *lens, const size_t *shifts, size_t nterms) {
    size_t m = 0;
    for (size_t t = 0; t < nterms; t++) m = std::max(m, shifts[t] + lens[t]);
    return m;
}
// the checks of a combination, before its workspace is taken and before its first launch: the size, every term's
// window inside [0, n), every term's destination row below nrows (rows == nullptr: every term in row 0) and the root
// (sa_ntt's SA_EROOTORDER / SA_ENOTPRIM).  Every offset is accepted, 0 included.
inline int coset_combine_check(int log_n, const size_t *lens, const size_t *shifts, const size_t *rows, size_t nrows,
                               size_t nterms, const uint64_t root[2]) {
    if (log_n < 1 || log_n > COSET_MAX_LOG) return SA_ESIZE;
    const size_t n = (size_t)1 << log_n;
    for (size_t t = 0; t < nterms; t++)
        if (shifts[t] > n || lens[t] > n - shifts[t] || (rows ? rows[t] : 0) >= nrows) return SA_ESIZE;
    return ntt_check_root(fe_to_mont(fe_from_limbs(root)), log_n);
}

// one row's: every term in row 0
inline int coset_combine_check(int log_n, const size_t *lens, const size_t *shifts, size_t nterms,
                               const uint64_t root[2]) {
    return coset_combine_check(log_n, lens, shifts, nullptr, 1, nterms, root);
}

// b.coset_combine: a backend's k_coset_combine over nrows rows.  A backend whose coset_combine takes one row, (out,
// g, pw, ncomb, log_n, first), serves nrows == 1.
template <class B>
auto coset_combine_call(B &b, fe *out, const CombineGroup &g, const fe *pw, long long ncomb, int log_n,
                        long long nrows, int first, int) -> decltype(b.coset_combine(out, g, pw, ncomb, log_n, nrows,
                                                                                     first)) {
    return b.coset_combine(out, g, pw, ncomb, log_n, nrows, first);
}
template <class B>
int coset_combine_call(B &b, fe *out, const CombineGroup &g, const fe *pw, long long ncomb, int log_n, long long nrows,
                       int first, long) {
    return nrows == 1 ? b.coset_combine(out, g, pw, ncomb, log_n, first) : SA_ESIZE;
}

// out[r] = ntt(c_r[i] * offset^i, zero padded to n) for r < nrows, c_r[i] = sum_t w_t * srcs[t][i - shifts[t]] over
// the terms of row r (rows[t] == r; rows == nullptr puts every term in row 0) with shifts[t] <= i < shifts[t] +
// lens[t] (fast_coset_evaluate of each row's combination at order n): offset^i for i < ncomb into pw (ncomb elements,
// the longest row's), then the terms in groups of COMBINE_TERMS, one launch each over all rows (the first writes all
// of out, the others add), then one batched transform of the nrows rows in place -- 1 + ceil(nterms / 64) launches
// plus the transform's, whatever nrows.  With ncomb == 0 (no term, or only empty ones at shift 0) out is zeros from
// the group launches alone: no table, no transform.  out must not overlap any source.  nrows >= 1.
template <class B>
int coset_combine_evaluate(B &b, fe *out, size_t nrows, int log_n, const uint64_t root[2], const uint64_t offset[2],
                           const fe *const *srcs, const size_t *lens, const size_t *shifts, const size_t *rows,
                           const uint64_t *weights, size_t nterms, fe *pw) {
    const long long ncomb = (long long)coset_combine_len(lens, shifts, nterms);
    if (ncomb) SA_TRY(b.pow_table(pw, fe_to_mont(fe_from_limbs(offset)), ncomb));
    for (size_t t0 = 0; t0 == 0 || t0 < nterms; t0 += COMBINE_TERMS) {
        CombineGroup g;
        g.count = (int)std::min((size_t)COMBINE_TERMS, nterms - t0);
        for (int k = 0; k < g.count; k++)
            g.t[k] = CombineTerm{srcs[t0 + k], (long long)lens[t0 + k], (long long)shifts[t0 + k],
                                 rows ? (long long)rows[t0 + k] : 0, fe_to_mont(fe_from_limbs(weights + 2 * (t0 + k)))};
        SA_TRY(coset_combine_call(b, out, g, pw, ncomb, log_n, (long long)nrows, t0 == 0, 0));
    }
    return ncomb ? b.ntt(out, out, log_n, root, 0, nrows) : SA_OK;
}

// one combination: nrows = 1 of the schedule above, every term in row 0
template <class B>
int coset_combine_evaluate(B &b, fe *out, int log_n, const uint64_t root[2], const uint64_t offset[2],
                           const fe *const *srcs, const size_t *lens, const size_t *shifts, const uint64_t *weights,
                           size_t nterms, fe *pw) {
    return coset_combine_evaluate(b, out, 1, log_n, root, offset, srcs, lens, shifts, nullptr, weights, nterms, pw);
}

}  // namespace sa
