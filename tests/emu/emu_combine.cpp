// tests/emu/emu_combine.cpp -- TEST INFRASTRUCTURE: the CPU emulation of emu_coset.cpp (included whole, so k_pow_table
// and sa_ntt are the same emulated code as the coset plans') plus coset combinations: the library's own check and
// schedule (coset.cuh: coset_combine_check, coset_combine_evaluate) over a backend whose k_coset_combine is a loop
// over coset_combine_elem.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_combine.so emu_combine.cpp
#include "emu_coset.cpp"

// EmuCoset plus k_coset_combine
struct EmuCombine : EmuCoset {
    int coset_combine(fe *out, const CombineGroup &g, const fe *pw_m, long long ncomb, int log_n, int first) {
        return each(1ll << log_n, [&](long long i) { coset_combine_elem(out, g, pw_m, ncomb, first, i); });
    }
};

extern "C" {

// sa_coset_combine_evaluate with host source rows.  out is overwritten with the stale pattern once the checks pass,
// so an element the first group fails to write shows up whatever the caller's buffer held.
int emu_coset_combine_evaluate(uint64_t *out, int log_n, const uint64_t *root, const uint64_t *offset,
                               const void *const *srcs, const size_t *lens, const size_t *shifts,
                               const uint64_t *weights, size_t nterms) {
    SA_TRY(coset_combine_check(log_n, lens, shifts, nterms, root));
    std::vector<fe> pw = stale_workspace(coset_combine_len(lens, shifts, nterms));
    const std::vector<fe> stale = stale_workspace((size_t)1 << log_n);
    memcpy(out, stale.data(), sizeof(fe) * stale.size());
    EmuCombine b;
    return coset_combine_evaluate(b, (fe *)out, log_n, root, offset, (const fe *const *)srcs, lens, shifts, weights,
                                  nterms, pw.data());
}

}  // extern "C"
