// boundary.cuh -- boundary quotients on a coset (fast_stark.py:92-106 without host polynomials): the per-element
// bodies of k_boundary_point and k_boundary_store, the plan layout, the checks and the host schedules of the plan
// build and the apply.  The library (poly.cu) runs the schedules with kernel launches, the CPU emulation
// (tests/emu/emu_boundary.cpp) with loops over the element functions.
//
// Register s has the trace polynomial T_s, the interpolant I_s of its boundary values and the zerofier Z_s of its
// boundary points.  With n = 2^log_n and x_i = offset * root^i an apply computes
//     codewords[s][i] = V_s(x_i) = (T_s(x_i) - I_s(x_i)) / Z_s(x_i),
//     quot[s][j]      = U_s[j] * offset^-j  (j < ncoef),   U_s = intt(V_s),
// and flags[s] != 0 when U_s has a non-zero coefficient at some j >= max(0, ncoef - deg Z_s).  With n >= ncoef and
// n > deg Z_s the division (T_s - I_s) / Z_s is exact if and only if that tail is zero: then U_s * Z_s and T_s - I_s
// both have degree below n and agree on n points.  An exact division's row is the reference's quotient followed by
// zeros and its codeword is fast_coset_evaluate's of the quotient, bit for bit.
//
// The schedules take the backend of coset.cuh plus b.upload(dst, host_src, count), b.download(host_dst, src, count),
// b.clear_flags(flags, count) (a memset in stream order), b.boundary_point (k_boundary_point) and b.boundary_store
// (k_boundary_store).
#pragma once
#include <algorithm>
#include <cstdint>

#include "coset.cuh"

namespace sa {

// ---- element functions ----
// cw[b][i] = (cw[b][i] - I_b(x_i)) * 1/Z_b(x_i): the transformed trace row minus the plan's interpolant value, times
// the plan's inverse zerofier value (ival canonical, izinv_m Montgomery form, both rows `stride` elements apart)
// (idx < batch * n)
SA_HD void boundary_point_elem(fe *cw, const fe *ival, const fe *izinv_m, long long stride, int log_n, long long idx) {
    const long long p = (idx >> log_n) * stride + (idx & ((1ll << log_n) - 1));
    tile_st(cw + idx, fe_montmul(fe_sub(tile_ld(cw + idx), tile_ld(ival + p)), tile_ld(izinv_m + p)));
}
// quot[b][j] = U[b][j] * offset^-j for j < ncoef (ipw_m = offset^-j in Montgomery form, U = ws); returns whether U[b][j]
// is a non-zero coefficient of the row's tail j >= ncoef - deg Z_b (deg = the plan's degree section), i.e. part of a
// remainder.  Indices from batch * n on, up to the warp's end, store nothing and return false.
SA_HD bool boundary_store_elem(fe *quot, const fe *ws, const fe *ipw_m, const fe *deg, long long ncoef, int log_n,
                               long long batch, long long idx) {
    if (idx >= batch << log_n) return false;
    const long long b = idx >> log_n, j = idx & ((1ll << log_n) - 1);
    const fe u = tile_ld(ws + idx), d = tile_ldg(deg + b);
    if (j < ncoef) tile_st(quot + b * ncoef + j, fe_montmul(u, tile_ld(ipw_m + j)));
    return j >= ncoef - ((long long)d.v[0] | (long long)d.v[1] << 32) && !fe_is_zero(u);
}
// Whether `lane` raises its row's flag, given the warp's ballot of boundary_store_elem: the lowest set lane among those
// of its row.  A warp covers 32 consecutive indices from a multiple of 32, so it lies in one row from n = 32 on and
// covers 32 / n whole rows below: one atomicOr per row a warp touches.
SA_HD bool boundary_flag_leader(uint32_t ballot, int lane, int log_n) {
    const uint32_t row = log_n >= 5 ? 0xFFFFFFFFu : ((1u << (1 << log_n)) - 1) << (lane & ~((1 << log_n) - 1));
    const uint32_t mine = ballot & row;
    return (mine & (0u - mine)) == (1u << lane);
}

// ---- plan layout ----
// A plan is a device buffer of boundary_plan_layout(log_n, nregs).elems elements, laid out by (log_n, nregs) alone;
// every section and every row starts on a 256-byte (16-element) boundary, S = sec16(n):
//   offset^i | offset^-i                              (2 S, Montgomery form)
//   1/Z_s(x_i), s < nregs                             (nregs S, Montgomery form)
//   I_s(x_i), s < nregs                               (nregs S, canonical)
//   deg Z_s, s < nregs (limbs 0 and 1 of an element)  (sec16(nregs))
// 32 n (1 + nregs) + 16 sec16(nregs) bytes from n = 16 on.  The plan keeps I_s(x_i) rather than I_s(x_i) / Z_s(x_i):
// the point kernel subtracts before it multiplies, still one product per point, and the build needs no product.
struct BoundaryPlan {
    int log_n = 0;
    long long n = 0, stride = 0;                           // stride = S, the distance of two rows of a section
    size_t pw = 0, ipw = 0, izinv = 0, ival = 0, deg = 0;  // element offsets of the sections
    size_t elems = 0;                                      // 0: no plan for these sizes
};
inline BoundaryPlan boundary_plan_layout(int log_n, size_t nregs) {
    BoundaryPlan L;
    if (log_n < 1 || log_n > COSET_MAX_LOG || nregs == 0) return L;
    const size_t S = sec16((size_t)1 << log_n);
    const unsigned __int128 r = nregs, elems = (2 + 2 * r) * S + ((r + 15) & ~(unsigned __int128)15);
    if (elems * sizeof(fe) > (unsigned __int128)SIZE_MAX) return L;
    L.log_n = log_n;
    L.n = 1ll << log_n;
    L.stride = (long long)S;
    L.ipw = S;
    L.izinv = 2 * S;
    L.ival = L.izinv + nregs * S;
    L.deg = L.ival + nregs * S;
    L.elems = (size_t)elems;
    return L;
}

// ---- checks, before any workspace is taken and before any launch ----
// a build's: the sizes (log_n 1..30, nregs >= 1 with a plan that fits size_t, every zlens[s] and ilens[s] 1..n), an
// offset other than 0 (the tail check needs n distinct points) and the root (SA_EROOTORDER / SA_ENOTPRIM)
inline int boundary_plan_check(int log_n, const size_t *zlens, const size_t *ilens, size_t nregs,
                               const uint64_t root[2], const uint64_t offset[2]) {
    if (boundary_plan_layout(log_n, nregs).elems == 0) return SA_ESIZE;
    const size_t n = (size_t)1 << log_n;
    for (size_t s = 0; s < nregs; s++)
        if (zlens[s] < 1 || zlens[s] > n || ilens[s] < 1 || ilens[s] > n) return SA_ESIZE;
    if (fe_is_zero(fe_to_mont(fe_from_limbs(offset)))) return SA_ESIZE;
    return ntt_check_root(fe_to_mont(fe_from_limbs(root)), log_n);
}
// an apply's: nregs >= 1 with a plan, ncoef 1..n and the root
inline int boundary_apply_check(int log_n, size_t nregs, size_t ncoef, const uint64_t root[2]) {
    if (boundary_plan_layout(log_n, nregs).elems == 0) return SA_ESIZE;
    return coset_check(log_n, ncoef, 1, root);
}
// a build's outcome once its work has completed: SA_ESIZE when a zerofier row's top coefficient (tops[s], downloaded
// by the build) is zero, since the tail check takes deg Z_s = zlens[s] - 1; else SA_EDIVZERO when some Z_s vanishes on
// the coset (the build's zero flag)
inline int boundary_plan_verdict(const fe *tops, size_t nregs, int zero_flag) {
    for (size_t s = 0; s < nregs; s++)
        if (fe_is_zero(tops[s])) return SA_ESIZE;
    return zero_flag ? SA_EDIVZERO : SA_OK;
}

// ---- host schedules ----
// The plan: offset^i and offset^-i, then per register Z_s's coset transform (k_coset_load + sa_ntt in ws, n elements)
// inverted into the plan by k_batch_inverse (a zero raises *flag), I_s's coset transform straight into the plan, and
// the download of Z_s's top coefficient into tops[s]; last the degrees zlens[s] - 1, staged in degs and uploaded.  The
// caller keeps tops and degs (nregs elements each) alive until the stream has completed, then takes
// boundary_plan_verdict.
template <class B>
int boundary_plan_build(B &b, fe *plan, const fe *const *zerofiers, const size_t *zlens, const fe *const *interpolants,
                        const size_t *ilens, size_t nregs, int log_n, const uint64_t root[2], const uint64_t offset[2],
                        fe *ws, int *flag, fe *tops, fe *degs) {
    const BoundaryPlan L = boundary_plan_layout(log_n, nregs);
    const fe off_m = fe_to_mont(fe_from_limbs(offset));
    SA_TRY(b.pow_table(plan + L.pw, off_m, L.n));
    SA_TRY(b.pow_table(plan + L.ipw, fe_mont_inv(off_m), L.n));
    for (size_t s = 0; s < nregs; s++) {
        fe *iz = plan + L.izinv + s * L.stride, *iv = plan + L.ival + s * L.stride;
        SA_TRY(b.coset_load(ws, zerofiers[s], plan + L.pw, (long long)zlens[s], log_n, 1));
        SA_TRY(b.ntt(ws, ws, log_n, root, 0, 1));
        SA_TRY(b.batch_inverse(iz, ws, L.n, flag));
        SA_TRY(b.coset_load(iv, interpolants[s], plan + L.pw, (long long)ilens[s], log_n, 1));
        SA_TRY(b.ntt(iv, iv, log_n, root, 0, 1));
        SA_TRY(b.download(tops + s, zerofiers[s] + zlens[s] - 1, 1));
        const uint64_t d = zlens[s] - 1;
        degs[s] = fe_make((uint32_t)d, (uint32_t)(d >> 32), 0, 0);
    }
    return b.upload(plan + L.deg, degs, nregs);
}

// The apply for trace[nregs][ncoef] (coefficient rows): quot[nregs][ncoef], codewords[nregs][n], flags[nregs].  The
// flags are cleared first; then per chunk of coset_batch_max(log_n) registers: the coset load into the codewords, one
// batched forward transform in place, k_boundary_point, one batched inverse transform from the codewords into ws and
// k_boundary_store -- five launches plus the transforms' per chunk, whatever its size.  ws = n elements per register
// of a chunk.
template <class B>
int boundary_quotients(B &b, fe *quot, fe *codewords, uint32_t *flags, const fe *plan, const fe *trace, size_t nregs,
                       size_t ncoef, int log_n, const uint64_t root[2], fe *ws) {
    const BoundaryPlan L = boundary_plan_layout(log_n, nregs);
    const size_t n = (size_t)L.n, chunk = std::min(nregs, coset_batch_max(log_n));
    SA_TRY(b.clear_flags(flags, nregs));
    for (size_t s0 = 0; s0 < nregs; s0 += chunk) {
        const size_t nb = std::min(chunk, nregs - s0);
        fe *cw = codewords + s0 * n;
        SA_TRY(b.coset_load(cw, trace + s0 * ncoef, plan + L.pw, (long long)ncoef, log_n, (long long)nb));
        SA_TRY(b.ntt(cw, cw, log_n, root, 0, nb));
        SA_TRY(b.boundary_point(cw, plan + L.ival + s0 * L.stride, plan + L.izinv + s0 * L.stride, L.stride, log_n,
                                (long long)nb));
        SA_TRY(b.ntt(ws, cw, log_n, root, 1, nb));
        SA_TRY(b.boundary_store(quot + s0 * ncoef, flags + s0, ws, plan + L.ipw, plan + L.deg + s0, (long long)ncoef,
                                log_n, (long long)nb));
    }
    return SA_OK;
}

}  // namespace sa
