// ntt_plan.cuh -- how an n-point transform (code/ntt.py:3-30) is cut into tile passes: the roots,
// the contents of the twiddle tables and the pass sequence.  The library (ntt.cu) runs it with
// kernel launches, the CPU emulation (tests/emu) with loops over the kernels' phase functions.
//
//   log_n <= 10 : one pass, every transform is one tile column.
//   log_n 11..20: four-step split n = n1 * n2 (n1 = 2^l1 >= n2 = 2^l2):
//       pass 1: for every column j2, an n1-point transform over j1 (stride n2),
//               times w^(k1*j2) [* n^-1 for intt], written to tmp[k1][j2];
//       pass 2: for every row k1 of tmp, an n2-point transform over j2,
//               written to out[k1 + n1*k2].
//     With j = j1*n2 + j2 and k = k1 + n1*k2:  w^(jk) = (w^n2)^(j1 k1) * w^(j2 k1) * (w^n1)^(j2 k2).
//   log_n 21..26: the same split applied twice, n = n1 * n2 * n3, j = j1*(n2 n3) + j2*n3 + j3,
//       k = k1 + n1*k2 + n1*n2*k3:
//       pass 1: n1-point transforms over j1 (stride n2 n3), times w^(k1*m), m = j2*n3 + j3;
//       pass 2: inside every k1 block, n2-point transforms over j2 (stride n3), times (w^n1)^(k2*j3);
//       pass 3: n3-point transforms over j3 (contiguous), written to out[k1 + n1*k2 + n1*n2*k3].
//   log_n 27..30: the same three passes, but the pass-1 matrix w^(k1*m) would have n entries (16 GiB at
//       2^30).  With m = j2*n3 + j3 it factors as (w^n3)^(k1*j2) * w^(k1*j3): pass 1 multiplies by one entry
//       of an n1 x n2 table A (which also carries n^-1 for intt) and one of an n1 x n3 table B.
#pragma once
#include <cstring>

#include "../../include/sa_b200.h"
#include "ntt_tile.cuh"

namespace sa {

// every digit of the three-pass split stays <= 10 (one tile) and every in-tile row offset below 2^31
constexpr int NTT_MAX_LOG_N = 30;
// largest size whose pass-1 twiddles are one n-entry matrix (1 GiB at 2^26); above it they are factored
constexpr int NTT_FULL_TWB_MAX_LOG_N = 26;

// Thread `thread` of a power table: out[slot(e)] = base^e * lead (Montgomery form) for its 16 consecutive
// exponents e < count.  swz != 0 stores in the bank-spreading order of tile_tw_slot (stage-twiddle tables,
// count % 64 == 0 or count < 8 so the permutation stays inside the table).
SA_HD void ntt_pow_table_thread(fe *out, const fe &base_m, const fe &lead_m, long long count, int swz,
                                long long thread) {
    const long long e0 = thread * 16;
    if (e0 >= count) return;
    fe acc = fe_montmul(fe_mont_pow_u64(base_m, (uint64_t)e0), lead_m);
    for (int i = 0; i < 16 && e0 + i < count; i++) {
        const long long e = e0 + i;
        tile_st(out + (swz ? (long long)tile_tw_slot((int)e) : e), acc);
        acc = fe_montmul(acc, base_m);
    }
}
// Thread `idx` of an n1 x n2 matrix: out[k * n2 + j] = w^(k*j) * scale (Montgomery form) for its 16
// consecutive j; row k is the power table of w^k
SA_HD void ntt_twb_table_thread(fe *out, const fe &w_m, const fe &scale_m, int n1, int n2, long long idx) {
    const long long per_row = (n2 + 15) / 16;
    const long long k = idx / per_row;
    const long long j0 = (idx % per_row) * 16;
    if (k >= n1) return;
    const fe wk = fe_mont_pow_u64(w_m, (uint64_t)k);
    fe acc = fe_montmul(fe_mont_pow_u64(wk, (uint64_t)j0), scale_m);
    for (int i = 0; i < 16 && j0 + i < n2; i++) {
        tile_st(out + k * n2 + j0 + i, acc);
        acc = fe_montmul(acc, wk);
    }
}

struct NttShape {
    int log_n, l1, l2, l3;  // l3 > 0: three passes
    int twb_split;          // three passes with the pass-1 matrix factored into A (n1 x n2) and B (n1 x n3)
};
// force3: 1 = split into three digits even when two would do, 2 = the same with factored pass-1 twiddles
// (tests exercise both three-pass plans at small sizes); 0 = the plan of the size
SA_HD NttShape ntt_shape(int log_n, int force3 = 0) {
    NttShape s;
    s.log_n = log_n;
    s.l3 = 0;
    s.twb_split = 0;
    if (log_n <= 10 && !force3) {
        s.l1 = log_n;
        s.l2 = 0;
    } else if (log_n <= 20 && !force3) {
        s.l2 = log_n / 2;
        s.l1 = log_n - s.l2;
    } else {
        s.l3 = log_n / 3;
        s.l1 = (log_n + 2) / 3;
        s.l2 = log_n - s.l1 - s.l3;
        s.twb_split = s.l3 > 0 && (log_n > NTT_FULL_TWB_MAX_LOG_N || force3 == 2) ? 1 : 0;
    }
    return s;
}

// cst[k] = w_Rmax^k (Montgomery), Rmax = min(16, L), where wL_m generates the L-point transform
inline void ntt_fill_cst(fe cst[8], const fe &wL_m, int L) {
    const int rmax = L >= 16 ? 16 : L;
    const fe wr = fe_mont_pow_u64(wL_m, (uint64_t)(L / rmax));
    fe acc = fe_mont_one();
    for (int k = 0; k < 8; k++) {
        cst[k] = (k < rmax / 2 || k == 0) ? acc : fe_mont_one();
        acc = fe_montmul(acc, wr);
    }
}

// single pass: `batch` contiguous transforms of n = 2^log_n elements, one tile column each
inline void ntt_fill_common(TileArgs &a) {
    a.in_sb2 = a.out_sb2 = 0;
    a.inner = 1;
    a.has_scale = 0;
    a.scale = fe_mont_one();
    a.twb = nullptr;
    a.twb_stride = 0;
    a.npeer = 0;
    a.mc_out = nullptr;
    a.twb_b = nullptr;
}
// three-pass split (see the header comment).  tmp: n * batch workspace; out doubles as the first
// intermediate (a tile reads all of its elements before it writes them, so in == out is fine).
// twb1_b != nullptr: factored pass-1 twiddles, twb1 = A (n1 x n2) and twb1_b = B (n1 x n3)
inline void ntt_fill_3pass_a(TileArgs &a, const fe *in, fe *mid, const NttShape &s, size_t batch, const fe *tw1,
                             const fe *twb1, const fe *twb1_b, const fe cst1[8]) {
    const long long n = 1ll << s.log_n, m = 1ll << (s.l2 + s.l3);
    ntt_fill_common(a);
    a.in = in; a.out = mid; a.tw = tw1;
    a.twb = twb1; a.twb_stride = m;
    if (twb1_b != nullptr) {  // columns m = j2 * n3 + j3: A has n2 columns, B the remaining n3 = m / n2
        a.twb_stride = 1ll << s.l2;
        a.twb_b = twb1_b;
    }
    a.in_sr = m; a.in_sc = 1; a.in_sb = n;
    a.out_sr = m; a.out_sc = 1; a.out_sb = n;
    a.ncols = (int)m; a.nbatch = (int)batch;
    for (int k = 0; k < 8; k++) a.cst[k] = cst1[k];
}
inline void ntt_fill_3pass_b(TileArgs &a, const fe *mid, fe *tmp, const NttShape &s, size_t batch, const fe *tw2,
                             const fe *twb2, const fe cst2[8]) {
    const long long n1 = 1ll << s.l1, n3 = 1ll << s.l3, m = 1ll << (s.l2 + s.l3);
    ntt_fill_common(a);
    a.in = mid; a.out = tmp; a.tw = tw2;
    a.twb = twb2; a.twb_stride = n3;
    a.in_sr = n3; a.in_sc = 1; a.in_sb = m;   // batch item = (b, k1): contiguous blocks of m
    a.out_sr = n3; a.out_sc = 1; a.out_sb = m;
    a.ncols = (int)n3; a.nbatch = (int)(batch * n1);
    for (int k = 0; k < 8; k++) a.cst[k] = cst2[k];
}
inline void ntt_fill_3pass_c(TileArgs &a, const fe *tmp, fe *out, const NttShape &s, size_t batch, const fe *tw3,
                             const fe cst3[8]) {
    const long long n = 1ll << s.log_n, n1 = 1ll << s.l1, n2 = 1ll << s.l2, n3 = 1ll << s.l3, m = n2 * n3;
    ntt_fill_common(a);
    a.in = tmp; a.out = out; a.tw = tw3;
    // batch item = (b, k2); column = k1 (adjacent k1 -> adjacent outputs); row = j3 / k3
    a.in_sr = 1; a.in_sc = m; a.in_sb = n; a.in_sb2 = n3;
    a.out_sr = n1 * n2; a.out_sc = 1; a.out_sb = n; a.out_sb2 = n1;
    a.inner = (int)n2;
    a.ncols = (int)n1; a.nbatch = (int)(batch * n2);
    for (int k = 0; k < 8; k++) a.cst[k] = cst3[k];
}

inline void ntt_fill_single(TileArgs &a, const fe *in, fe *out, int log_n, size_t batch, const fe *tw,
                            const fe cst[8], int has_scale, const fe &scale_m) {
    const long long n = 1ll << log_n;
    ntt_fill_common(a);
    a.in = in;
    a.out = out;
    a.tw = tw;
    a.twb = nullptr;
    a.twb_stride = 0;
    a.in_sr = 1; a.in_sc = n; a.in_sb = 0;
    a.out_sr = 1; a.out_sc = n; a.out_sb = 0;
    a.ncols = (int)batch;
    a.nbatch = 1;
    a.has_scale = has_scale;
    a.scale = scale_m;
    for (int k = 0; k < 8; k++) a.cst[k] = cst[k];
}
inline void ntt_fill_pass1(TileArgs &a, const fe *in, fe *tmp, const NttShape &s, size_t batch, const fe *tw1,
                           const fe *twb, const fe cst1[8]) {
    const long long n = 1ll << s.log_n, n2 = 1ll << s.l2;
    ntt_fill_common(a);
    a.in = in;
    a.out = tmp;
    a.tw = tw1;
    a.twb = twb;
    a.twb_stride = n2;
    a.in_sr = n2; a.in_sc = 1; a.in_sb = n;
    a.out_sr = n2; a.out_sc = 1; a.out_sb = n;
    a.ncols = (int)n2;
    a.nbatch = (int)batch;
    a.has_scale = 0;
    a.scale = fe_mont_one();
    for (int k = 0; k < 8; k++) a.cst[k] = cst1[k];
}
inline void ntt_fill_pass2(TileArgs &a, const fe *tmp, fe *out, const NttShape &s, size_t batch, const fe *tw2,
                           const fe cst2[8]) {
    const long long n = 1ll << s.log_n, n1 = 1ll << s.l1, n2 = 1ll << s.l2;
    ntt_fill_common(a);
    a.in = tmp;
    a.out = out;
    a.tw = tw2;
    a.twb = nullptr;
    a.twb_stride = 0;
    a.in_sr = 1; a.in_sc = n2; a.in_sb = n;      // column = k1 (a row of tmp), row = j2
    a.out_sr = n1; a.out_sc = 1; a.out_sb = n;   // out[k1 + n1 * k2]
    a.ncols = (int)n1;
    a.nbatch = (int)batch;
    a.has_scale = 0;
    a.scale = fe_mont_one();
    for (int k = 0; k < 8; k++) a.cst[k] = cst2[k];
}

// validates the root like ntt.py:10-11: root_m (Montgomery form) must have order exactly n = 2^log_n
inline int ntt_check_root(const fe &root_m, int log_n) {
    const uint64_t n = 1ull << log_n;
    if (!fe_eq(fe_mont_pow_u64(root_m, n), fe_mont_one())) return SA_EROOTORDER;
    if (fe_eq(fe_mont_pow_u64(root_m, n / 2), fe_mont_one())) return SA_ENOTPRIM;
    return SA_OK;
}

// roots of the passes of one transform (Montgomery form)
struct NttRoots {
    fe w;           // the transform root: root itself, or root^-1 for intt (ntt.py:29)
    fe w1, w2, w3;  // roots of the pass-1, pass-2 and pass-3 transforms (one pass: w1 = w)
    fe wsub;        // three passes: root of the length n2*n3 sub-transforms, base of the pass-2 matrix
    fe scale;       // n^-1 for intt (ntt.py:27), else 1: in the pass-1 matrix, or applied by a single pass
};
inline NttRoots ntt_roots(const NttShape &s, const fe &root_m, int inverse) {
    NttRoots r;
    r.w = inverse ? fe_mont_inv(root_m) : root_m;
    r.scale = inverse ? fe_mont_inv(fe_to_mont(fe_from_u64(1ull << s.log_n))) : fe_mont_one();
    r.w1 = r.w;
    r.w2 = r.w3 = r.wsub = fe_mont_one();
    if (s.l3 > 0) {
        r.w1 = fe_mont_pow_u64(r.w, 1ull << (s.l2 + s.l3));  // n1-point transforms over j1
        r.wsub = fe_mont_pow_u64(r.w, 1ull << s.l1);
        r.w2 = fe_mont_pow_u64(r.wsub, 1ull << s.l3);         // n2-point transforms over j2
        r.w3 = fe_mont_pow_u64(r.wsub, 1ull << s.l2);         // n3-point transforms over j3
    } else if (s.l2 > 0) {
        r.w1 = fe_mont_pow_u64(r.w, 1ull << s.l2);  // root of the length-n1 column transforms
        r.w2 = fe_mont_pow_u64(r.w, 1ull << s.l1);  // root of the length-n2 row transforms
    }
    return r;
}

// the tables and constants of one transform's passes
struct NttTables {
    fe *tw1 = nullptr, *tw2 = nullptr, *tw3 = nullptr;  // stage twiddles of the pass-1, -2, -3 transforms
    fe *twb = nullptr, *twb2 = nullptr;                 // matrices applied by pass 1 and pass 2
    fe *twb_b = nullptr;  // factored pass-1 twiddles (twb_split): twb = A, twb_b = B
    fe cst1[8], cst2[8], cst3[8];
    fe scale_m;  // single pass: n^-1 (Montgomery) for intt
    int has_scale = 0;
};

// Builds the tables of a transform of shape s.  pow(&table, base_m, count) makes a stage-twiddle table
// (ntt_pow_table_thread, lead 1, tile_tw_slot order), twb(&table, w_m, scale_m, rows, cols) a matrix
// (ntt_twb_table_thread); both return SA_OK or an error code.
template <class Pow, class Twb>
int ntt_build_tables(NttTables &t, const NttShape &s, const fe &root_m, int inverse, Pow &&pow, Twb &&twb) {
    const NttRoots r = ntt_roots(s, root_m, inverse);
    const int n1 = 1 << s.l1, n2 = 1 << s.l2, n3 = 1 << s.l3;
    int rc;
    if ((rc = pow(&t.tw1, r.w1, n1)) != SA_OK) return rc;
    ntt_fill_cst(t.cst1, r.w1, n1);
    if (s.l2 == 0) {
        t.has_scale = inverse ? 1 : 0;
        t.scale_m = r.scale;
        return SA_OK;
    }
    if ((rc = pow(&t.tw2, r.w2, n2)) != SA_OK) return rc;
    ntt_fill_cst(t.cst2, r.w2, n2);
    if (s.l3 == 0) return twb(&t.twb, r.w, r.scale, n1, (long long)n2);
    if ((rc = pow(&t.tw3, r.w3, n3)) != SA_OK) return rc;
    ntt_fill_cst(t.cst3, r.w3, n3);
    if (s.twb_split) {
        // A[k1][j2] = (w^n3)^(k1*j2) * scale, B[k1][j3] = w^(k1*j3): A * B = w^(k1*(j2*n3 + j3)) * scale
        if ((rc = twb(&t.twb, fe_mont_pow_u64(r.w, (uint64_t)n3), r.scale, n1, (long long)n2)) != SA_OK) return rc;
        if ((rc = twb(&t.twb_b, r.w, fe_mont_one(), n1, (long long)n3)) != SA_OK) return rc;
    } else if ((rc = twb(&t.twb, r.w, r.scale, n1, (long long)n2 * n3)) != SA_OK) {
        return rc;
    }
    return twb(&t.twb2, r.wsub, fe_mont_one(), n2, (long long)n3);
}

// Runs the passes of a transform of shape s: in -> out through tmp (n * batch elements, unused by a single
// pass; three passes use out as their first intermediate, which is fine when in == out because a tile reads
// all of its elements before it writes them).  run(logl, a, last) runs one pass of logl-point tile
// transforms and returns SA_OK or an error code; `last` marks the pass that writes out.
template <class Run>
int ntt_run_passes(const NttShape &s, const NttTables &t, const fe *in, fe *out, fe *tmp, size_t batch, Run &&run) {
    TileArgs a;
    memset(&a, 0, sizeof(a));
    int rc;
    if (s.l2 == 0) {
        ntt_fill_single(a, in, out, s.log_n, batch, t.tw1, t.cst1, t.has_scale, t.scale_m);
        return run(s.log_n, a, true);
    }
    if (s.l3 > 0) {
        ntt_fill_3pass_a(a, in, out, s, batch, t.tw1, t.twb, t.twb_b, t.cst1);
        if ((rc = run(s.l1, a, false)) != SA_OK) return rc;
        ntt_fill_3pass_b(a, out, tmp, s, batch, t.tw2, t.twb2, t.cst2);
        if ((rc = run(s.l2, a, false)) != SA_OK) return rc;
        ntt_fill_3pass_c(a, tmp, out, s, batch, t.tw3, t.cst3);
        return run(s.l3, a, true);
    }
    ntt_fill_pass1(a, in, tmp, s, batch, t.tw1, t.twb, t.cst1);
    if ((rc = run(s.l1, a, false)) != SA_OK) return rc;
    ntt_fill_pass2(a, tmp, out, s, batch, t.tw2, t.cst2);
    return run(s.l2, a, true);
}

}  // namespace sa
