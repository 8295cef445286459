// verify.cuh -- the data-parallel checks of FastStark.verify and Stark.verify (fast_stark.py:180-286, stark.py:172-275,
// fri.py:132-231) for many proofs: Merkle paths, FRI colinearity, the combination at the opened indices and the last
// codeword's degree.  __host__ __device__ element functions (verify.cu runs one per thread, tests/emu/emu_verify.cpp
// runs them in loops) and the checks the C ABI makes before any launch.  Every flag is 0 where the check passes.
#pragma once
#include <cstdint>

#include "air.cuh"   // air_pow, the compiled AIR program (AIR_FIRST / AIR_LAST records)
#include "hash.cuh"  // the leaf and node digests

namespace sa {

// ---- Merkle.verify (merkle.py:28-43) ----
// The leaf's digest is blake2b of its decimal ASCII; level l hashes (cur || sibling) when bit l of the index is 0 and
// (sibling || cur) when it is 1, the index read least significant bit first; the last digest is compared with the
// root.  An index at or above 2^depth (the reference's "cannot verify invalid index") and a depth above 63 fail.
SA_HD uint32_t merkle_verify_elem(const uint64_t *roots, const fe *leaves, const uint64_t *leaf_index,
                                  const uint32_t *depth, const uint64_t *paths, const uint64_t *path_offset,
                                  long long i) {
    const uint32_t d = depth[i];
    uint64_t idx = leaf_index[i];
    if (d > 63 || (idx >> d) != 0) return 1;
    uint64_t h[8];
    merkle_leaf_digest(h, leaves[i]);
    const uint64_t *sib = paths + 8 * path_offset[i];
    for (uint32_t l = 0; l < d; l++, idx >>= 1, sib += 8) {
        if (idx & 1)
            merkle_node_digest(h, sib, h);
        else
            merkle_node_digest(h, h, sib);
    }
    const uint64_t *root = roots + 8 * i;
    uint64_t diff = 0;
    for (int w = 0; w < 8; w++) diff |= h[w] ^ root[w];
    return diff != 0;
}

// ---- test_colinearity (univariate.py:156-160) as the reference computes it ----
// Polynomial.interpolate_domain over (x0, y0), (x1, y1), (x2, y2) is sum_i c_i prod_{j != i} (X - x_j) with
// c_i = y_i prod_{j != i} inverse(x_i - x_j), where inverse(0) = 0 (xgcd, algebra.py:87-89).  Its X^2 coefficient is
// c0 + c1 + c2 and its X coefficient -(c0 (x1 + x2) + c1 (x0 + x2) + c2 (x0 + x1)); the degree is 1 exactly when
// the first is zero and the second is not.  So three points on a constant line (degree 0) fail, and alpha equal to
// ax or bx zeroes two of the c_i and leaves a quadratic or a constant: it fails too.  Canonical in; 1 = not
// colinear.
SA_HD uint32_t lagrange_colinear(const fe &x0, const fe &y0, const fe &x1, const fe &y1, const fe &x2, const fe &y2) {
    const fe i01 = fe_mont_inv(fe_to_mont(fe_sub(x0, x1)));  // Montgomery inverses of the differences
    const fe i02 = fe_mont_inv(fe_to_mont(fe_sub(x0, x2)));
    const fe i12 = fe_mont_inv(fe_to_mont(fe_sub(x1, x2)));
    // canonical y times two Montgomery inverses: canonical c_i (inverse(x_j - x_i) = -inverse(x_i - x_j))
    const fe c0 = fe_montmul(fe_montmul(y0, i01), i02);
    const fe c1 = fe_neg(fe_montmul(fe_montmul(y1, i01), i12));
    const fe c2 = fe_montmul(fe_montmul(y2, i02), i12);
    const fe quad = fe_add(fe_add(c0, c1), c2);
    const fe lin = fe_add(fe_add(fe_mul(c0, fe_add(x1, x2)), fe_mul(c1, fe_add(x0, x2))), fe_mul(c2, fe_add(x0, x1)));
    return !(fe_is_zero(quad) && !fe_is_zero(lin));
}

// FRI round r's check at a-index a (fri.py:204-207): ax = offset^(2^r) omega^(2^r a), bx = offset^(2^r)
// omega^(2^r (a + n / 2^(r+1))) = -ax, cx = alpha.  offset_m and omega_m are the first round's, in Montgomery form.
SA_HD uint32_t fri_colinear_elem(const fe *ay, const fe *by, const fe *cy, const uint64_t *a_index, const fe *alpha,
                                 const uint32_t *round, const fe &offset_m, const fe &omega_m, long long i) {
    fe off = offset_m, om = omega_m;
    for (uint32_t r = 0; r < round[i]; r++) {
        off = fe_montmul(off, off);
        om = fe_montmul(om, om);
    }
    const fe ax = fe_from_mont(fe_montmul(off, fe_mont_pow_u64(om, a_index[i])));
    return lagrange_colinear(ax, ay[i], fe_neg(ax), by[i], alpha[i], cy[i]);
}

// ---- one AIR at one point: the compiled program of air.cuh walked once ----
// emit(c, N_c(point)) for every constraint c < ncons in order, N_c canonical; x_m and the nregs current and nregs
// next trace values cur_m / nxt_m in Montgomery form.  A constraint without records is 0 (an MPolynomial without
// terms evaluates to zero).  The walk is air_eval_elem's with the point's values in place of a coset row's.
template <class Emit>
SA_HD void air_point_elem(const fe *prog, const fe &x_m, const fe *cur_m, const fe *nxt_m, long long ncons, int nregs,
                          Emit &&emit) {
    const fe h0 = prog[0];
    const long long nrec = (long long)h0.v[0] | (long long)h0.v[1] << 32, stride = 2 + (nregs + 1) / 2;
    long long c_at = 0;
    fe acc = fe_zero(), s = fe_zero(), xp = fe_mont_one();
    for (long long t = 0; t < nrec; t++) {
        const fe *rec = prog + 1 + t * stride;
        const fe h = rec[0];
        const long long c = h.v[0];
        if (c >= ncons) break;
        for (; c_at < c; c_at++, acc = fe_zero()) emit(c_at, acc);
        if (h.v[1] & AIR_FIRST) {
            xp = air_pow(x_m, h.v[2]);
            s = fe_zero();
        } else {
            xp = fe_montmul(xp, air_pow(x_m, h.v[2]));
        }
        s = fe_add(s, fe_montmul(rec[1], xp));
        if (h.v[1] & AIR_LAST) {
            for (int w = 0; w < (nregs + 1) / 2; w++) {
                const fe e4 = rec[2 + w];
                for (int k = 0; k < 4; k++) {
                    const int v = 4 * w + k;
                    if (v < 2 * nregs && e4.v[k]) s = fe_montmul(s, air_pow(v < nregs ? cur_m[v] : nxt_m[v - nregs], e4.v[k]));
                }
            }
            acc = fe_add(acc, s);
        }
    }
    for (; c_at < ncons; c_at++, acc = fe_zero()) emit(c_at, acc);
}

// ---- the combination at one opened index (fast_stark.py:244-284, stark.py:222-272) ----
// Item layout, verify_item(nregs) elements: [0] the FRI index i (limb 0), [1] FRI's opened value there, [2, 2 + nregs)
// the boundary quotient leaves at i, [2 + nregs, 2 + 2 nregs) those at (i + ef) mod n, [2 + 2 nregs] the randomizer
// leaf at i, [3 + 2 nregs] the transition zerofier leaf at i (read only without zerofier coefficients).
// Proof layout, verify_proof(nregs, ncons, blen) elements: the W = 1 + 2 ncons + 2 nregs weights, the ncons
// transition shifts and nregs boundary shifts (limb 0 each, below 2^32), then per register its boundary zerofier's
// and its interpolant's coefficients, blen each (low to high, zero padded).  Items k q .. k q + k - 1 are proof q's.
SA_HD long long verify_item(long long nregs) { return 4 + 2 * nregs; }
SA_HD long long verify_proof(long long nregs, long long ncons, long long blen) {
    return 1 + 2 * ncons + 2 * nregs + ncons + nregs + 2 * nregs * blen;
}
constexpr int VERIFY_MAX_REGS = 16;  // the trace values of one point live in per-thread arrays of this size

// Horner with canonical coefficients and x in Montgomery form: the canonical value
SA_HD fe horner_elem(const fe *coef, long long len, const fe &x_m) {
    fe acc = fe_zero();
    for (long long j = len - 1; j >= 0; j--) acc = fe_add(fe_montmul(acc, x_m), coef[j]);
    return acc;
}

// 0 when the combination equals FRI's value, 1 when it does not, 2 when the transition zerofier is zero at x (the
// reference's division raises "divide by zero" there).  zcoef (zlen coefficients, canonical) is the plain Stark's
// transition zerofier; NULL takes the item's zerofier leaf (FastStark).
SA_HD uint32_t verify_combination_elem(const fe *items, const fe *proofs, long long k, const fe *prog, long long ncons,
                                       int nregs, long long blen, const fe *zcoef, long long zlen, const fe &offset_m,
                                       const fe &omega_m, int log_n, long long ef, long long j) {
    const fe *it = items + j * verify_item(nregs);
    const fe *pr = proofs + (j / k) * verify_proof(nregs, ncons, blen);
    const long long W = 1 + 2 * ncons + 2 * nregs;
    const fe *w = pr, *shifts = pr + W, *bc = pr + W + ncons + nregs;
    const uint64_t mask = ((uint64_t)1 << log_n) - 1, i = it[0].v[0] | (uint64_t)it[0].v[1] << 32;
    const fe x_m = fe_montmul(offset_m, fe_mont_pow_u64(omega_m, i & mask));
    const fe xn_m = fe_montmul(offset_m, fe_mont_pow_u64(omega_m, (i + (uint64_t)ef) & mask));
    fe cur_m[VERIFY_MAX_REGS], nxt_m[VERIFY_MAX_REGS];
    fe acc = fe_montmul(w[0], fe_to_mont(it[2 + 2 * nregs]));  // the randomizer's term
    for (int s = 0; s < nregs; s++) {
        const fe *zs = bc + 2 * s * blen, *is = zs + blen;
        const fe leaf = it[2 + s], leafn = it[2 + nregs + s];
        cur_m[s] = fe_to_mont(fe_add(fe_mul(leaf, horner_elem(zs, blen, x_m)), horner_elem(is, blen, x_m)));
        nxt_m[s] = fe_to_mont(fe_add(fe_mul(leafn, horner_elem(zs, blen, xn_m)), horner_elem(is, blen, xn_m)));
        // bqv (w + w' x^shift)
        const fe t = fe_add(w[W - 2 * nregs + 2 * s],
                            fe_montmul(w[W - 2 * nregs + 2 * s + 1], air_pow(x_m, shifts[ncons + s].v[0])));
        acc = fe_add(acc, fe_mul(leaf, t));
    }
    const fe z = zcoef ? horner_elem(zcoef, zlen, x_m) : it[3 + 2 * nregs];
    if (fe_is_zero(z)) return 2;
    const fe zinv_m = fe_mont_inv(fe_to_mont(z));
    air_point_elem(prog, x_m, cur_m, nxt_m, ncons, nregs, [&](long long c, const fe &tcv) {
        const fe q = fe_montmul(tcv, zinv_m);  // canonical quotient
        const fe t = fe_add(w[1 + 2 * c], fe_montmul(w[2 + 2 * c], air_pow(x_m, shifts[c].v[0])));
        acc = fe_add(acc, fe_mul(q, t));
    });
    return !fe_eq(acc, it[1]);
}

// ---- the last codeword's degree (fri.py:151-174) ----
// the highest j < n with coeffs[row n + j] != 0, or -1: the degree of the interpolant of the row (the inverse
// transform's coefficients scaled by offset^-j, which keeps every zero where it is).  The kernel takes the maximum
// over a row's elements with an atomic; this is one element's contribution.
SA_HD long long degree_elem(const fe *coeffs, int log_n, long long idx) {
    return fe_is_zero(coeffs[idx]) ? -1 : (idx & ((1ll << log_n) - 1));
}

// ---- checks, before any launch ----
constexpr unsigned long long VERIFY_LIMIT = 1ULL << 59;
inline int verify_count_check(size_t count) { return count >= VERIFY_LIMIT ? SA_ESIZE : SA_OK; }
inline int verify_combination_check(size_t k, size_t nproofs, size_t ncons, size_t nregs, size_t blen, size_t zlen,
                                    bool have_z, int log_n, size_t ef) {
    if (nregs == 0 || nregs > (size_t)VERIFY_MAX_REGS || ncons == 0 || ncons >= ((size_t)1 << 32) || blen == 0 ||
        blen >= ((size_t)1 << 32) || log_n < 1 || log_n > 30 || ef >= ((size_t)1 << log_n))
        return SA_ESIZE;
    if (have_z && (zlen == 0 || zlen >= VERIFY_LIMIT)) return SA_ESIZE;
    unsigned long long items;
    if (__builtin_mul_overflow((unsigned long long)k, (unsigned long long)nproofs, &items) || items >= VERIFY_LIMIT)
        return SA_ESIZE;
    if ((unsigned long long)verify_proof((long long)nregs, (long long)ncons, (long long)blen) * nproofs >= VERIFY_LIMIT ||
        items * (unsigned long long)verify_item((long long)nregs) >= VERIFY_LIMIT)
        return SA_ESIZE;
    return SA_OK;
}

}  // namespace sa
