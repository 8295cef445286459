// tests/emu/emu_air.cpp -- TEST INFRASTRUCTURE: the CPU emulation of emu_coset.cpp (included whole, so the coset
// division plan, k_pow_table, the coset loads and stores and sa_ntt are the same emulated code as the coset plans')
// plus transition quotients: the library's own checks, compilation and schedules (air.cuh: air_plan_check,
// air_compile, air_plan_build, air_apply_check, air_quotients) over a backend whose k_air_eval is a loop over
// air_eval_elem.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_air.so emu_air.cpp
#include "emu_coset.cpp"

#include "../../stark-anatomy_b200/csrc/air.cuh"

// EmuCoset plus k_pow_table with a lead, the program's upload and k_air_eval
struct EmuAir : EmuCoset {
    int pow_table_lead(fe *out, const fe &base_m, const fe &lead_m, long long count) {
        return each((count + 15) / 16, [&](long long t) { ntt_pow_table_thread(out, base_m, lead_m, count, 0, t); });
    }
    int upload(fe *dst, const fe *src, size_t n) {
        memcpy(dst, src, sizeof(fe) * n);
        return SA_OK;
    }
    int air_eval(fe *V, const fe *prog, const fe *x_m, const fe *iz_m, const fe *ext, long long c0, long long nb,
                 int nregs, int log_n) {
        return each(1ll << log_n, [&](long long i) { air_eval_elem(V, prog, x_m, iz_m, ext, c0, nb, nregs, log_n, i); });
    }
};

extern "C" {

size_t emu_air_plan_bytes(int log_n, size_t max_ncoef, size_t nregs, size_t nterms) {
    return sizeof(fe) * air_plan_layout(log_n, max_ncoef, nregs, nterms).elems;
}
// sa_air_plan with a host zerofier and plan; the zerofier's codeword starts from the stale pattern
int emu_air_plan(uint64_t *plan, const uint64_t *coeffs, const uint32_t *exps, const size_t *term_start, size_t ncons,
                 size_t nregs, size_t max_ncoef, const uint64_t *zerofier, size_t zlen, int log_n,
                 const uint64_t *root, const uint64_t *offset, const uint64_t *step) {
    SA_TRY(air_plan_check(log_n, exps, term_start, ncons, nregs, max_ncoef, zlen, root));
    const std::vector<fe> prog = air_compile(coeffs, exps, term_start, ncons, nregs);
    std::vector<fe> ws = stale_workspace((size_t)1 << log_n);
    int flag = 0;
    EmuAir b;
    SA_TRY(air_plan_build(b, (fe *)plan, prog, (const fe *)zerofier, zlen, log_n, root, offset, step, ws.data(),
                          &flag));
    return flag ? SA_EDIVZERO : SA_OK;
}
// sa_air_quotients with host rows.  The workspace and out start from the stale pattern once the checks pass, so an
// element the schedule fails to write shows up whatever the caller's buffer held.
int emu_air_quotients(uint64_t *out, const uint64_t *plan, const uint64_t *trace, size_t nregs, size_t ncoef,
                      size_t qlen, size_t ncons, int log_n, const uint64_t *root) {
    SA_TRY(air_apply_check(log_n, nregs, ncoef, qlen, ncons, root));
    std::vector<fe> ws = stale_workspace(air_ws_elems(nregs, ncons, log_n));
    const std::vector<fe> stale = stale_workspace(ncons * qlen);
    memcpy(out, stale.data(), sizeof(fe) * stale.size());
    EmuAir b;
    return air_quotients(b, (fe *)out, (const fe *)plan, (const fe *)trace, nregs, ncoef, qlen, ncons, log_n, root,
                         ws.data());
}

}  // extern "C"
