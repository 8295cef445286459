// tests/emu/emu_coset.cpp -- TEST INFRASTRUCTURE: the CPU emulation of emu.cpp (included whole, so sa_ntt's
// emulation and the subproduct tree's backend are the same code) plus coset division plans, their batched apply
// and batched coset evaluation: the library's own checks and schedules (coset.cuh) over a backend whose kernels
// are loops over their element functions.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_coset.so emu_coset.cpp
#include "emu.cpp"

#include "../../stark-anatomy_b200/csrc/coset.cuh"

// EmuTree plus the kernels of the coset schedules: k_pow_table (lead 1, natural order), k_coset_load / _quot / _store
struct EmuCoset : EmuTree {
    int pow_table(fe *out, const fe &base_m, long long count) {
        return each((count + 15) / 16, [&](long long t) { ntt_pow_table_thread(out, base_m, fe_mont_one(), count, 0, t); });
    }
    int coset_load(fe *ws, const fe *lhs, const fe *pw_m, long long ncoef, int log_n, long long batch) {
        return each(batch << log_n, [&](long long i) { coset_load_elem(ws, lhs, pw_m, ncoef, log_n, i); });
    }
    int coset_quot(fe *ws, const fe *inv_m, int log_n, long long batch) {
        return each(batch << log_n, [&](long long i) { coset_quot_elem(ws, inv_m, log_n, i); });
    }
    int coset_store(fe *out, const fe *ws, const fe *ipw_m, long long qlen, int log_n, long long batch) {
        return each(batch << log_n, [&](long long i) { coset_store_elem(out, ws, ipw_m, qlen, log_n, i); });
    }
};

// The workspaces start out holding what an earlier call left (here: a non-zero pattern), as the library's do, so a
// kernel that fails to write an element it owns shows up.
static std::vector<fe> stale_workspace(size_t n) { return std::vector<fe>(n, fe_make(0x5a5a5a5au, 1, 2, 3)); }

extern "C" {

size_t emu_coset_div_plan_bytes(int log_n) { return sizeof(fe) * coset_div_plan_layout(log_n).elems; }
int emu_coset_div_plan(uint64_t *plan, const uint64_t *divisor, size_t dlen, int log_n, const uint64_t *root,
                       const uint64_t *offset) {
    SA_TRY(coset_div_plan_check(log_n, dlen, root, offset));
    std::vector<fe> ws = stale_workspace((size_t)1 << log_n);
    int flag = 0;
    EmuCoset b;
    SA_TRY(coset_div_plan_build(b, (fe *)plan, (const fe *)divisor, dlen, log_n, root, offset, ws.data(), &flag));
    return flag ? SA_EDIVZERO : SA_OK;
}
int emu_coset_div_apply_batch(uint64_t *out, const uint64_t *plan, const uint64_t *lhs, size_t ncoef, size_t qlen,
                              int log_n, const uint64_t *root, size_t batch) {
    SA_TRY(coset_check(log_n, ncoef, qlen, root));
    std::vector<fe> ws = stale_workspace(((size_t)1 << log_n) * std::min(batch, coset_batch_max(log_n)));
    EmuCoset b;
    return coset_div_apply(b, (fe *)out, (const fe *)plan, (const fe *)lhs, ncoef, qlen, log_n, root, batch, ws.data());
}
int emu_coset_evaluate_batch(uint64_t *out, const uint64_t *coeffs, size_t ncoef, int log_n, const uint64_t *root,
                             const uint64_t *offset, size_t batch) {
    SA_TRY(coset_check(log_n, ncoef, 1, root));
    std::vector<fe> pw = stale_workspace(ncoef);
    EmuCoset b;
    return coset_evaluate(b, (fe *)out, (const fe *)coeffs, ncoef, log_n, root, offset, batch, pw.data());
}

}  // extern "C"
