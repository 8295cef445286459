// tests/emu/emu_boundary.cpp -- TEST INFRASTRUCTURE: the CPU emulation of emu_coset.cpp (included whole, so
// k_pow_table, the coset loads, k_batch_inverse and sa_ntt are the same emulated code as the coset plans') plus
// boundary quotients: the library's own checks and schedules (boundary.cuh: boundary_plan_check,
// boundary_plan_build, boundary_plan_verdict, boundary_apply_check, boundary_quotients) over a backend whose
// k_boundary_point is a loop over boundary_point_elem and whose k_boundary_store runs warps of 32 indices: each
// lane's boundary_store_elem, the warp's ballot, then boundary_flag_leader's lanes raise their row's flag.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_boundary.so emu_boundary.cpp
#include "emu_coset.cpp"

#include "../../stark-anatomy_b200/csrc/boundary.cuh"

// EmuCoset plus the copies, the flags' memset and the two boundary kernels
struct EmuBoundary : EmuCoset {
    int upload(fe *dst, const fe *src, size_t n) {
        memcpy(dst, src, sizeof(fe) * n);
        return SA_OK;
    }
    int download(fe *dst, const fe *src, size_t n) { return upload(dst, src, n); }
    int clear_flags(uint32_t *flags, size_t n) {
        memset(flags, 0, sizeof(uint32_t) * n);
        return SA_OK;
    }
    int boundary_point(fe *cw, const fe *ival, const fe *izinv_m, long long stride, int log_n, long long batch) {
        return each(batch << log_n, [&](long long i) { boundary_point_elem(cw, ival, izinv_m, stride, log_n, i); });
    }
    int boundary_store(fe *quot, uint32_t *flags, const fe *ws, const fe *ipw_m, const fe *deg, long long ncoef,
                       int log_n, long long batch) {
        for (long long w = 0; w < batch << log_n; w += 32) {
            uint32_t ballot = 0;
            for (int lane = 0; lane < 32; lane++)
                if (boundary_store_elem(quot, ws, ipw_m, deg, ncoef, log_n, batch, w + lane)) ballot |= 1u << lane;
            for (int lane = 0; lane < 32; lane++)
                if ((ballot >> lane & 1u) && boundary_flag_leader(ballot, lane, log_n)) {
                    flags[(w + lane) >> log_n] |= 1u;
                    store_atomics++;
                }
        }
        return SA_OK;
    }
    long long store_atomics = 0;
};

// the atomicOr count of the last emulated apply's stores (one per flagged row a warp touches)
static long long g_store_atomics = 0;

extern "C" {

size_t emu_boundary_plan_bytes(int log_n, size_t nregs) { return sizeof(fe) * boundary_plan_layout(log_n, nregs).elems; }
// sa_boundary_plan with host rows and plan; the zerofier's codeword starts from the stale pattern
int emu_boundary_plan(uint64_t *plan, const uint64_t *const *zerofiers, const size_t *zlens,
                      const uint64_t *const *interpolants, const size_t *ilens, size_t nregs, int log_n,
                      const uint64_t *root, const uint64_t *offset) {
    SA_TRY(boundary_plan_check(log_n, zlens, ilens, nregs, root, offset));
    std::vector<fe> ws = stale_workspace((size_t)1 << log_n), tops(nregs), degs(nregs);
    int flag = 0;
    EmuBoundary b;
    SA_TRY(boundary_plan_build(b, (fe *)plan, (const fe *const *)zerofiers, zlens, (const fe *const *)interpolants,
                               ilens, nregs, log_n, root, offset, ws.data(), &flag, tops.data(), degs.data()));
    return boundary_plan_verdict(tops.data(), nregs, flag);
}
// sa_boundary_quotients with host rows.  The workspace, quot, codewords and flags start from a stale pattern once the
// checks pass, so an element the schedule fails to write, or a flag it fails to clear, shows up whatever the caller's
// buffers held.
int emu_boundary_quotients(uint64_t *quot, uint64_t *codewords, uint32_t *flags, const uint64_t *plan,
                           const uint64_t *trace, size_t nregs, size_t ncoef, int log_n, const uint64_t *root) {
    SA_TRY(boundary_apply_check(log_n, nregs, ncoef, root));
    const size_t n = (size_t)1 << log_n;
    std::vector<fe> ws = stale_workspace(n * std::min(nregs, coset_batch_max(log_n)));
    const std::vector<fe> sq = stale_workspace(nregs * ncoef), sc = stale_workspace(nregs * n);
    memcpy(quot, sq.data(), sizeof(fe) * sq.size());
    memcpy(codewords, sc.data(), sizeof(fe) * sc.size());
    for (size_t s = 0; s < nregs; s++) flags[s] = 0x5a5a5a5au;
    EmuBoundary b;
    const int rc = boundary_quotients(b, (fe *)quot, (fe *)codewords, flags, (const fe *)plan, (const fe *)trace, nregs,
                                      ncoef, log_n, root, ws.data());
    g_store_atomics = b.store_atomics;
    return rc;
}
long long emu_boundary_store_atomics() { return g_store_atomics; }

}  // extern "C"
