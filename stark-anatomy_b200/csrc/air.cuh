// air.cuh -- transition quotients of an AIR on a coset (fast_stark.py:108-113 without evaluate_symbolic): the
// per-point body of k_air_eval, the plan layout, the checks, the host-side compilation of the constraints and the
// host schedules of the plan build and the apply.  The library (poly.cu) runs the schedules with kernel launches, the
// CPU emulation (tests/emu/emu_air.cpp) with loops over the element functions.
//
// The constraints are polynomials in nvars = 1 + 2 nregs variables, FastStark's point: x, the trace rows T_s(x) and
// the next rows T_s(step * x).  With n = 2^log_n, x_i = offset * root^i and N_c(x) = C_c(x, T(x), T(step * x)), row c
// of an apply is
//     out[c][j] = U_c[j] * offset^-j  (j < qlen),   U_c = intt(N_c(x_i) / Z(x_i)),
// the coset division of coset.cuh with the numerator's values computed point by point instead of transformed from
// its coefficients.  Where every term's degree bound e_0 + (e_1 + ... + e_2nregs) (max_ncoef - 1) is below n (the
// build checks it) N_c has degree < n, so its values determine it and the rows are fast_coset_divide's at order n,
// bit for bit, clean division or not.
//
// The exact apply adds a remainder check: flags[c] = 0 exactly when U_c[j] = 0 for every tail <= j < n.  With
// tail = n - deg Z that is the reference's test of N_c / Z (univariate.py:50-53) for every numerator, N_c = 0 and
// deg N_c < deg Z included: the build keeps deg N_c < n, so if U_c vanishes from n - deg Z on, U_c Z has degree below
// n and agrees with N_c on the n points x_i, hence Z divides N_c; conversely an exact quotient has degree
// deg N_c - deg Z < n - deg Z, and N_c / Z = U_c on the coset.
//
// An apply takes a batch of traces, trace[batch][nregs][ncoef] -> out[batch][ncons][qlen]: row b * ncons + c is
// constraint c of trace b, the row the apply of trace b alone gives.  A batch shares the launches of one apply within
// a chunk (air_chunks below); the single-trace apply is batch 1.
//
// The schedules take the backend of coset.cuh plus b.pow_table_lead(out, base_m, lead_m, count) (k_pow_table with a
// lead), b.upload(dst, host_src, count) and b.air_eval (k_air_eval, air_eval_rows_elem); the exact apply also
// b.clear_flags(flags, count) (a memset in stream order) and b.air_store_exact (k_air_store_exact).
#pragma once
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <vector>

#include "boundary.cuh"  // boundary_flag_leader, shared by the exact store
#include "coset.cuh"

namespace sa {

// ---- the compiled program ----
// Element 0 holds the record count (limbs 0, 1).  Record t is AIR_REC(nregs) elements:
//   [0] header: v[0] = constraint, v[1] = AIR_FIRST | AIR_LAST flags, v[2] = x-exponent step, v[3] = 0
//   [1] the coefficient (canonical)
//   [2 ..] the group's trace exponents e_1 .. e_2nregs, four per element
// Records run in constraint order; within a constraint the terms sharing one trace-exponent vector form a group, in
// ascending x exponent.  The first record of a group steps from x^0, every other from the previous record's x power:
// dense x-polynomials cost one product per term, a sparse high power O(log) products.
constexpr uint32_t AIR_FIRST = 1, AIR_LAST = 2;
inline size_t air_rec(size_t nregs) { return 2 + (nregs + 1) / 2; }

// b^e, b and the result in Montgomery form, left to right from b itself: e == 1 costs no product, e == 0 gives 1
SA_HD fe air_pow(const fe &b_m, uint32_t e) {
    if (e == 0) return fe_mont_one();
    int top = 31;
    while (!((e >> top) & 1u)) top--;
    fe acc = b_m;
    for (int bit = top - 1; bit >= 0; bit--) {
        acc = fe_montmul(acc, acc);
        if ((e >> bit) & 1u) acc = fe_montmul(acc, b_m);
    }
    return acc;
}

// ---- element functions: the body of k_air_eval for one point ----
// V[c - c0][i] = N_c(x_i) / Z(x_i) for the constraints c0 <= c < c0 + nb of one trace, walking the program once:
// records of other constraints are skipped, a constraint without records gets zeros.  x_m and iz_m are the plan's x_i
// and 1/Z_i, cur and nxt the trace's nregs rows T_s(x_i) and nregs rows T_s(step * x_i) (canonical); coefficients are
// canonical, so a coefficient times a Montgomery-form power is canonical again  (i < n)
SA_HD void air_eval_elem(fe *V, const fe *prog, const fe *x_m, const fe *iz_m, const fe *cur, const fe *nxt,
                         long long c0, long long nb, int nregs, int log_n, long long i) {
    const long long n = 1ll << log_n;
    const fe x = tile_ld(x_m + i), iz = tile_ld(iz_m + i), h0 = tile_ldg(prog);
    const long long nrec = (long long)h0.v[0] | (long long)h0.v[1] << 32, stride = 2 + (nregs + 1) / 2;
    long long c_at = c0;
    fe acc = fe_zero(), s = fe_zero(), xp = fe_mont_one();
    for (long long t = 0; t < nrec; t++) {
        const fe *rec = prog + 1 + t * stride;
        const fe h = tile_ldg(rec);
        const long long c = h.v[0];
        if (c < c0) continue;
        if (c >= c0 + nb) break;
        for (; c_at < c; c_at++, acc = fe_zero()) tile_st(V + (c_at - c0) * n + i, fe_montmul(acc, iz));
        if (h.v[1] & AIR_FIRST) {
            xp = air_pow(x, h.v[2]);
            s = fe_zero();
        } else {
            xp = fe_montmul(xp, air_pow(x, h.v[2]));
        }
        s = fe_add(s, fe_montmul(tile_ldg(rec + 1), xp));
        if (h.v[1] & AIR_LAST) {
            for (int w = 0; w < (nregs + 1) / 2; w++) {
                const fe e4 = tile_ldg(rec + 2 + w);
                for (int k = 0; k < 4; k++) {
                    const int v = 4 * w + k;
                    if (v < 2 * nregs && e4.v[k]) {
                        const fe *row = v < nregs ? cur + v * n : nxt + (v - nregs) * n;
                        s = fe_montmul(s, air_pow(fe_to_mont(tile_ld(row + i)), e4.v[k]));
                    }
                }
            }
            acc = fe_add(acc, s);
        }
    }
    for (; c_at < c0 + nb; c_at++, acc = fe_zero()) tile_st(V + (c_at - c0) * n + i, fe_montmul(acc, iz));
}
// the same for one trace whose 2 nregs rows lie together: current rows at ext, next rows at ext + nregs n
SA_HD void air_eval_elem(fe *V, const fe *prog, const fe *x_m, const fe *iz_m, const fe *ext, long long c0,
                         long long nb, int nregs, int log_n, long long i) {
    air_eval_elem(V, prog, x_m, iz_m, ext, ext + ((long long)nregs << log_n), c0, nb, nregs, log_n, i);
}
// The rows r0 <= r < r0 + nb of a chunk of bp traces, row r = b * ncons + c being trace b's constraint c:
// air_eval_elem once per trace the rows touch, trace b's current rows at ext + b nregs n and its next rows at
// ext + (bp + b) nregs n (the chunk's two coset loads, each of bp * nregs rows)  (i < n)
SA_HD void air_eval_rows_elem(fe *V, const fe *prog, const fe *x_m, const fe *iz_m, const fe *ext, long long r0,
                              long long nb, long long ncons, long long bp, int nregs, int log_n, long long i) {
    const long long n = 1ll << log_n, rows = (long long)nregs * n;
    for (long long b = r0 / ncons; b * ncons < r0 + nb; b++) {
        const long long lo = r0 > b * ncons ? r0 : b * ncons;
        const long long hi = r0 + nb < (b + 1) * ncons ? r0 + nb : (b + 1) * ncons;
        air_eval_elem(V + (lo - r0) * n, prog, x_m, iz_m, ext + b * rows, ext + (bp + b) * rows, lo - b * ncons,
                      hi - lo, nregs, log_n, i);
    }
}

// ---- element function: the body of k_air_store_exact ----
// coset_store_elem's store of row b = idx >> log_n (out[b][j] = U[b][j] * offset^-j for j < qlen, U = ws) and whether
// U[b][j] is a non-zero coefficient at j >= tail, i.e. part of a remainder; the rows are coset_store_elem's bit for
// bit.  Indices from batch * n on, up to the warp's end, store nothing and return false: the kernel's ballot then
// raises each row's flag once per warp with boundary_flag_leader.
SA_HD bool air_store_exact_elem(fe *out, const fe *ws, const fe *ipw_m, long long qlen, long long tail, int log_n,
                                long long batch, long long idx) {
    if (idx >= batch << log_n) return false;
    const long long b = idx >> log_n, j = idx & ((1ll << log_n) - 1);
    const fe u = tile_ld(ws + idx);
    if (j < qlen) tile_st(out + b * qlen + j, fe_montmul(u, tile_ld(ipw_m + j)));
    return j >= tail && !fe_is_zero(u);
}

// ---- plan layout ----
// A plan is a device buffer of air_plan_layout(...).elems elements; every section starts on a 256-byte (16-element)
// boundary, S = sec16(n):
//   offset^i | 1/Z_i | offset^-i   (the coset division plan of the zerofier, 3 S)
//   (offset * step)^j, j < n       (S; the next rows' load)
//   x_i = offset * root^i          (S)
//   the program                    (sec16(1 + nterms * air_rec(nregs)))
// all field sections in Montgomery form.  Every section but the program sits where log_n alone puts it, so an apply
// finds them from (log_n, nregs) -- the arguments it has -- and the kernel reads the program's length from the plan.
// 80 n + 16 sec16(1 + nterms (2 + ceil(nregs / 2))) bytes from n = 16 on.
struct AirPlan {
    int log_n = 0;
    long long n = 0;
    CosetPlan div;
    size_t spw = 0, x = 0, prog = 0;  // element offsets of the sections after the division plan
    size_t elems = 0;                 // 0: no plan for these sizes
};
constexpr size_t AIR_MAX_TERMS = (size_t)1 << 32;
inline AirPlan air_plan_layout(int log_n, size_t max_ncoef, size_t nregs, size_t nterms) {
    AirPlan L;
    const CosetPlan d = coset_div_plan_layout(log_n);
    if (d.elems == 0 || nregs == 0 || nregs > AIR_MAX_TERMS || max_ncoef < 1 || max_ncoef > (size_t)d.n ||
        nterms >= AIR_MAX_TERMS)
        return L;
    L.log_n = log_n;
    L.n = d.n;
    L.div = d;
    L.spw = d.elems;
    L.x = L.spw + sec16((size_t)L.n);
    L.prog = L.x + sec16((size_t)L.n);
    L.elems = L.prog + sec16(1 + nterms * air_rec(nregs));
    return L;
}

// A batched apply runs in chunks of whole traces, and within a chunk in row chunks of the chunk's bp * ncons
// constraint rows.  A chunk takes 2 nregs transformed rows per trace and n elements per row of a row chunk: 16 bytes
// per element of its own workspace and 16 of the transform's, 32 n bytes per row, as coset_batch_max counts them.  So
// a chunk holds as many traces as keep its 2 nregs + ncons rows per trace within coset_batch_max(log_n) rows (1 GiB),
// at least one, and a row chunk at most coset_batch_max(log_n) rows: a chunk of several traces is then one row chunk
// and issues the launches of one trace's apply, and a batch of one is chunked as the single apply always was.
struct AirChunks {
    size_t traces = 0, rows = 0;
};
inline size_t air_chunk(size_t ncons, int log_n) { return std::min(ncons, coset_batch_max(log_n)); }
inline size_t air_batch_max(size_t nregs, size_t ncons, int log_n) {
    const size_t cap = coset_batch_max(log_n), per = 2 * nregs + ncons;
    return cap == 0 ? 0 : std::max<size_t>(1, cap / per);
}
inline AirChunks air_chunks(size_t nregs, size_t ncons, size_t batch, int log_n) {
    AirChunks k;
    k.traces = std::max<size_t>(1, std::min(batch, air_batch_max(nregs, ncons, log_n)));
    k.rows = air_chunk(k.traces * ncons, log_n);
    return k;
}
inline size_t air_ws_elems(size_t nregs, const AirChunks &k, int log_n) {
    return ((size_t)1 << log_n) * (2 * nregs * k.traces + k.rows);
}
inline size_t air_ws_elems(size_t nregs, size_t ncons, int log_n) {
    return air_ws_elems(nregs, air_chunks(nregs, ncons, 1, log_n), log_n);
}

// ---- checks, before any workspace is taken and before any launch ----
// a build's: the sizes (log_n 1..30, nregs and ncons >= 1, max_ncoef and zlen 1..n), term_start non-decreasing, every
// term's degree bound below n (pointwise evaluation is exact there) and the root (SA_EROOTORDER / SA_ENOTPRIM)
inline int air_plan_check(int log_n, const uint32_t *exps, const size_t *term_start, size_t ncons, size_t nregs,
                          size_t max_ncoef, size_t zlen, const uint64_t root[2]) {
    if (log_n < 1 || log_n > COSET_MAX_LOG || nregs == 0 || ncons == 0) return SA_ESIZE;
    const uint64_t n = (uint64_t)1 << log_n;
    if (max_ncoef < 1 || max_ncoef > n || zlen < 1 || zlen > n) return SA_ESIZE;
    for (size_t c = 0; c < ncons; c++)
        if (term_start[c + 1] < term_start[c]) return SA_ESIZE;
    if (air_plan_layout(log_n, max_ncoef, nregs, term_start[ncons]).elems == 0) return SA_ESIZE;
    const size_t nvars = 1 + 2 * nregs;
    for (size_t t = term_start[0]; t < term_start[ncons]; t++) {
        const uint32_t *e = exps + t * nvars;
        if (e[0] >= n) return SA_ESIZE;
        uint64_t tdeg = 0;
        for (size_t v = 1; v < nvars; v++) tdeg += e[v];
        // e_0 + tdeg (max_ncoef - 1) < n, without overflow
        if (max_ncoef > 1 && tdeg > (n - 1 - e[0]) / (max_ncoef - 1)) return SA_ESIZE;
    }
    return ntt_check_root(fe_to_mont(fe_from_limbs(root)), log_n);
}
// an apply's: the sizes (ncoef and qlen 1..n) and the root
inline int air_apply_check(int log_n, size_t nregs, size_t ncoef, size_t qlen, size_t ncons, const uint64_t root[2]) {
    if (nregs == 0 || ncons == 0) return SA_ESIZE;
    return coset_check(log_n, ncoef, qlen, root);
}
// the exact apply's: the apply's, and tail 0..n
inline int air_exact_check(int log_n, size_t nregs, size_t ncoef, size_t qlen, size_t ncons, size_t tail,
                           const uint64_t root[2]) {
    SA_TRY(air_apply_check(log_n, nregs, ncoef, qlen, ncons, root));
    return tail > ((size_t)1 << log_n) ? SA_ESIZE : SA_OK;
}

// ---- compilation (host) ----
// the program of the terms term_start[0] .. term_start[ncons): the terms of each constraint sorted by (trace
// exponents, x exponent), grouped by trace exponents, x steps taken within a group
inline std::vector<fe> air_compile(const uint64_t *coeffs, const uint32_t *exps, const size_t *term_start, size_t ncons,
                                   size_t nregs) {
    const size_t nvars = 1 + 2 * nregs, rec = air_rec(nregs), nterms = term_start[ncons] - term_start[0];
    std::vector<fe> prog(1 + nterms * rec, fe_zero());
    prog[0] = fe_make((uint32_t)nterms, (uint32_t)((uint64_t)nterms >> 32), 0, 0);
    auto same_trace = [&](size_t a, size_t b) {
        return std::equal(exps + a * nvars + 1, exps + (a + 1) * nvars, exps + b * nvars + 1);
    };
    size_t r = 0;
    for (size_t c = 0; c < ncons; c++) {
        std::vector<size_t> ts(term_start[c + 1] - term_start[c]);
        std::iota(ts.begin(), ts.end(), term_start[c]);
        std::stable_sort(ts.begin(), ts.end(), [&](size_t a, size_t b) {
            return std::lexicographical_compare(exps + a * nvars + 1, exps + (a + 1) * nvars, exps + b * nvars + 1,
                                                exps + (b + 1) * nvars) ||
                   (same_trace(a, b) && exps[a * nvars] < exps[b * nvars]);
        });
        for (size_t k = 0; k < ts.size(); k++, r++) {
            const size_t t = ts[k];
            const bool first = k == 0 || !same_trace(ts[k - 1], t);
            const bool last = k + 1 == ts.size() || !same_trace(t, ts[k + 1]);
            const uint32_t dx = first ? exps[t * nvars] : exps[t * nvars] - exps[ts[k - 1] * nvars];
            fe *p = prog.data() + 1 + r * rec;
            p[0] = fe_make((uint32_t)c, (first ? AIR_FIRST : 0) | (last ? AIR_LAST : 0), dx, 0);
            p[1] = fe_from_limbs(coeffs + 2 * t);
            for (size_t v = 0; v < 2 * nregs; v++) p[2 + v / 4].v[v % 4] = exps[t * nvars + 1 + v];
        }
    }
    return prog;
}

// ---- host schedules ----
// The plan: the zerofier's coset division plan (coset_div_plan_build, ws = n elements), (offset * step)^j, x_i and
// the program compiled on the host and uploaded.  The caller reads *flag after the build (SA_EDIVZERO when Z vanishes
// on the coset) and keeps `prog` alive until the upload has completed.
template <class B>
int air_plan_build(B &b, fe *plan, const std::vector<fe> &prog, const fe *zerofier, size_t zlen, int log_n,
                   const uint64_t root[2], const uint64_t offset[2], const uint64_t step[2], fe *ws, int *flag) {
    const AirPlan L = air_plan_layout(log_n, 1, 1, 0);
    SA_TRY(coset_div_plan_build(b, plan, zerofier, zlen, log_n, root, offset, ws, flag));
    const fe off_m = fe_to_mont(fe_from_limbs(offset));
    SA_TRY(b.pow_table(plan + L.spw, fe_montmul(off_m, fe_to_mont(fe_from_limbs(step))), L.n));
    SA_TRY(b.pow_table_lead(plan + L.x, fe_to_mont(fe_from_limbs(root)), off_m, L.n));
    return b.upload(plan + L.prog, prog.data(), prog.size());
}

// The quotients of the plan's constraints for `batch` traces trace[batch][nregs][ncoef] (coefficient rows):
// out[batch][ncons][qlen], trace b's rows exactly the apply of trace b alone.  Per chunk of k.traces traces: the
// current rows of its traces loaded with offset^i and the next rows with (offset * step)^j, one batched forward
// transform of the 2 nregs rows per trace, then per row chunk of k.rows constraint rows k_air_eval, one batched
// inverse transform and store(r, nb, V), the store of rows r .. r + nb of out from V: 3 + 3 ceil(ncons / k.rows)
// launches per chunk plus the transforms', whatever nregs and the chunk's size.  ws = air_ws_elems(nregs, k, log_n)
// elements.  The library takes k = air_chunks(...); the emulation may take smaller chunks.
// b.air_eval: a backend's k_air_eval over the rows of a chunk of bp traces (air_eval_rows_elem).  A backend whose
// air_eval takes one trace's rows, (V, prog, x, iz, ext, c0, nb, nregs, log_n) as air_eval_elem does, serves chunks
// of one trace, the only chunks a batch of one makes.
template <class B>
auto air_eval_call(B &b, fe *V, const fe *prog, const fe *x, const fe *iz, const fe *ext, long long r0, long long nb,
                   long long ncons, long long bp, int nregs, int log_n, int)
    -> decltype(b.air_eval(V, prog, x, iz, ext, r0, nb, ncons, bp, nregs, log_n)) {
    return b.air_eval(V, prog, x, iz, ext, r0, nb, ncons, bp, nregs, log_n);
}
template <class B>
int air_eval_call(B &b, fe *V, const fe *prog, const fe *x, const fe *iz, const fe *ext, long long r0, long long nb,
                  long long /*ncons*/, long long bp, int nregs, int log_n, long) {
    return bp == 1 ? b.air_eval(V, prog, x, iz, ext, r0, nb, nregs, log_n) : SA_ESIZE;
}

template <class B, class Store>
int air_apply(B &b, const fe *plan, const fe *trace, size_t nregs, size_t ncoef, size_t ncons, size_t batch,
              int log_n, const uint64_t root[2], fe *ws, const AirChunks &k, Store store) {
    const AirPlan L = air_plan_layout(log_n, 1, nregs, 0);
    const size_t n = (size_t)L.n;
    for (size_t p0 = 0; p0 < batch; p0 += k.traces) {
        const size_t bp = std::min(k.traces, batch - p0), rows = bp * ncons;
        const fe *tr = trace + p0 * nregs * ncoef;
        fe *ext = ws, *V = ws + 2 * nregs * bp * n;
        SA_TRY(b.coset_load(ext, tr, plan + L.div.pw, (long long)ncoef, log_n, (long long)(bp * nregs)));
        SA_TRY(b.coset_load(ext + bp * nregs * n, tr, plan + L.spw, (long long)ncoef, log_n, (long long)(bp * nregs)));
        SA_TRY(b.ntt(ext, ext, log_n, root, 0, 2 * bp * nregs));
        for (size_t r0 = 0; r0 < rows; r0 += k.rows) {
            const size_t nb = std::min(k.rows, rows - r0);
            SA_TRY(air_eval_call(b, V, plan + L.prog, plan + L.x, plan + L.div.inv, ext, (long long)r0,
                                 (long long)nb, (long long)ncons, (long long)bp, (int)nregs, log_n, 0));
            SA_TRY(b.ntt(V, V, log_n, root, 1, nb));
            SA_TRY(store(p0 * ncons + r0, nb, V));
        }
    }
    return SA_OK;
}
// the apply: k_coset_store per row chunk
template <class B>
int air_quotients(B &b, fe *out, const fe *plan, const fe *trace, size_t nregs, size_t ncoef, size_t qlen,
                  size_t ncons, size_t batch, int log_n, const uint64_t root[2], fe *ws, const AirChunks &k) {
    const fe *ipw = plan + air_plan_layout(log_n, 1, nregs, 0).div.ipw;
    return air_apply(b, plan, trace, nregs, ncoef, ncons, batch, log_n, root, ws, k,
                     [&](size_t r, size_t nb, const fe *V) {
                         return b.coset_store(out + r * qlen, V, ipw, (long long)qlen, log_n, (long long)nb);
                     });
}
// the exact apply: the flags[batch][ncons] cleared first, then k_air_store_exact per row chunk -- the apply's
// launches plus one
template <class B>
int air_quotients_exact(B &b, fe *out, uint32_t *flags, const fe *plan, const fe *trace, size_t nregs, size_t ncoef,
                        size_t qlen, size_t ncons, size_t batch, size_t tail, int log_n, const uint64_t root[2],
                        fe *ws, const AirChunks &k) {
    const fe *ipw = plan + air_plan_layout(log_n, 1, nregs, 0).div.ipw;
    SA_TRY(b.clear_flags(flags, batch * ncons));
    return air_apply(b, plan, trace, nregs, ncoef, ncons, batch, log_n, root, ws, k,
                     [&](size_t r, size_t nb, const fe *V) {
                         return b.air_store_exact(out + r * qlen, flags + r, V, ipw, (long long)qlen, (long long)tail,
                                                  log_n, (long long)nb);
                     });
}

// the single-trace applies: batch 1 of the schedules above, with the library's chunks
template <class B>
int air_quotients(B &b, fe *out, const fe *plan, const fe *trace, size_t nregs, size_t ncoef, size_t qlen,
                  size_t ncons, int log_n, const uint64_t root[2], fe *ws) {
    return air_quotients(b, out, plan, trace, nregs, ncoef, qlen, ncons, 1, log_n, root, ws,
                         air_chunks(nregs, ncons, 1, log_n));
}
template <class B>
int air_quotients_exact(B &b, fe *out, uint32_t *flags, const fe *plan, const fe *trace, size_t nregs, size_t ncoef,
                        size_t qlen, size_t ncons, size_t tail, int log_n, const uint64_t root[2], fe *ws) {
    return air_quotients_exact(b, out, flags, plan, trace, nregs, ncoef, qlen, ncons, 1, tail, log_n, root, ws,
                               air_chunks(nregs, ncons, 1, log_n));
}

}  // namespace sa
