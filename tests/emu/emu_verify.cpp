// tests/emu/emu_verify.cpp -- TEST INFRASTRUCTURE: the CPU emulation of the verifier's element functions
// (csrc/verify.cuh): Merkle paths, the colinearity test, the AIR at one point and the combination, run item by item
// as the kernels run them thread by thread, plus the C ABI's checks.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_verify.so emu_verify.cpp
#include <cstring>
#include <vector>

#include "../../stark-anatomy_b200/csrc/verify.cuh"

using namespace sa;

extern "C" {

// flags[i] = merkle_verify_elem(..., i) for i < count (roots: 64 bytes per path, paths: 64-byte digests)
void emu_merkle_verify(uint32_t *flags, const void *roots, const void *leaves, const uint64_t *leaf_index,
                       const uint32_t *depth, const void *paths, const uint64_t *path_offset, long long count) {
    for (long long i = 0; i < count; i++)
        flags[i] = merkle_verify_elem((const uint64_t *)roots, (const fe *)leaves, leaf_index, depth,
                                      (const uint64_t *)paths, path_offset, i);
}

// lagrange_colinear over count triples of points, xs and ys (3 canonical elements each per item)
void emu_colinear(uint32_t *flags, const void *xs, const void *ys, long long count) {
    const fe *x = (const fe *)xs, *y = (const fe *)ys;
    for (long long i = 0; i < count; i++)
        flags[i] = lagrange_colinear(x[3 * i], y[3 * i], x[3 * i + 1], y[3 * i + 1], x[3 * i + 2], y[3 * i + 2]);
}

// fri_colinear_elem over count items
void emu_fri_colinear(uint32_t *flags, const void *ay, const void *by, const void *cy, const uint64_t *a_index,
                      const void *alpha, const uint32_t *round, const uint64_t offset[2], const uint64_t omega[2],
                      long long count) {
    const fe off = fe_to_mont(fe_from_limbs(offset)), om = fe_to_mont(fe_from_limbs(omega));
    for (long long i = 0; i < count; i++)
        flags[i] = fri_colinear_elem((const fe *)ay, (const fe *)by, (const fe *)cy, a_index, (const fe *)alpha, round,
                                     off, om, i);
}

// the AIR's constraint values at `count` points (point p: 1 + 2 nregs canonical elements) -> out[p][ncons],
// the constraints compiled by air_compile as sa_air_program compiles them
int emu_air_point(void *out, const uint64_t *coeffs, const uint32_t *exps, const size_t *term_start, size_t ncons,
                  size_t nregs, const void *points, long long count) {
    if (nregs == 0 || nregs > (size_t)VERIFY_MAX_REGS || ncons == 0) return SA_ESIZE;
    const std::vector<fe> prog = air_compile(coeffs, exps, term_start, ncons, nregs);
    const fe *pt = (const fe *)points;
    fe *o = (fe *)out;
    for (long long p = 0; p < count; p++) {
        const fe *q = pt + p * (1 + 2 * (long long)nregs);
        fe cur[VERIFY_MAX_REGS], nxt[VERIFY_MAX_REGS];
        for (size_t s = 0; s < nregs; s++) {
            cur[s] = fe_to_mont(q[1 + s]);
            nxt[s] = fe_to_mont(q[1 + nregs + s]);
        }
        air_point_elem(prog.data(), fe_to_mont(q[0]), cur, nxt, (long long)ncons, (int)nregs,
                       [&](long long c, const fe &v) { o[p * (long long)ncons + c] = v; });
    }
    return SA_OK;
}

// sa_verify_combination's checks, then verify_combination_elem over every item; the program compiled here
int emu_verify_combination(uint32_t *flags, const void *items, const void *proofs, size_t k, size_t nproofs,
                           const uint64_t *coeffs, const uint32_t *exps, const size_t *term_start, size_t ncons,
                           size_t nregs, size_t blen, const void *zcoef, size_t zlen, const uint64_t offset[2],
                           const uint64_t omega[2], int log_n, size_t ef) {
    SA_TRY(verify_combination_check(k, nproofs, ncons, nregs, blen, zlen, zcoef != nullptr, log_n, ef));
    const std::vector<fe> prog = air_compile(coeffs, exps, term_start, ncons, nregs);
    const fe off = fe_to_mont(fe_from_limbs(offset)), om = fe_to_mont(fe_from_limbs(omega));
    for (long long j = 0; j < (long long)(k * nproofs); j++)
        flags[j] = verify_combination_elem((const fe *)items, (const fe *)proofs, (long long)k, prog.data(),
                                           (long long)ncons, (int)nregs, (long long)blen, (const fe *)zcoef,
                                           (long long)zlen, off, om, log_n, (long long)ef, j);
    return SA_OK;
}

}  // extern "C"
